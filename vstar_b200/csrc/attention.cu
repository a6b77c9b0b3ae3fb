// Attention kernels.
//
//  vsb_flash_attn_bf16  : softmax(Q K^T * scale [+ causal]) V for head_dim 64 / 128, bf16 in/out, fp32
//                         online softmax.  Used by CLIP-L/14 (S=257, 16 heads x 64), OWL-ViT-B/16 (S=2305,
//                         12 x 64) and the 7B prefill/decode (32 x 128, causal, KV cache).  Reference op
//                         sites H2/H5/H10 (SURVEY.md §2b): transformers/models/clip/modeling_clip.py:261-329,
//                         transformers/models/llama/modeling_llama.py:199-221 (softmax in fp32, P cast to bf16).
//                         Round-1 implementation: FA2-style tiling (64 queries x 64 keys per step, cp.async
//                         double-buffered K/V in XOR-swizzled shared memory, ldmatrix + mma.sync.m16n8k16).
//                         The wgmma kernel of attention_tc.cu takes the shapes with Sq >= 64; attention is
//                         ~5 % of the per-crop FLOPs (BASELINE.md §3).
//  vsb_attn_small_bf16  : tiny-head attention of the SAM two-way transformer (head_dim 16 / 32, 6 tokens
//                         <-> 2304 image tokens); CUDA-core kernel, fp32 math.
//                         (/root/reference/VisualSearch/model/segment_anything/modeling/transformer.py:220-242)
#include <type_traits>

#include "common.cuh"
#include "vstar_b200.h"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
#define VSB_MMA_16816(TY)                                                                                                    \
  asm volatile(                                                                                                              \
      "mma.sync.aligned.m16n8k16.row.col.f32." TY "." TY ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"         \
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])                                                                      \
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1))
template <typename T>
__device__ __forceinline__ void mma_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  if constexpr (ElemT<T>::is_f16) VSB_MMA_16816(VSB_PTX_F16);
  else VSB_MMA_16816(VSB_PTX_BF16);
}

struct AttnParams {
  const void* q; const void* k; const void* v; void* o;     // element type T of the kernel (bf16 / f16)
  long long q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs;   // batch / row strides in elements; head h at +h*D
  int B, H, Sq, Sk;
  int causal;      // query i attends keys j <= i + (Sk - Sq)
  float scale_log2;
  const int* k_start = nullptr;   // decode kernel only: first valid key of each batch entry (left-padded ragged batches)
  // segment mask (mma.sync kernel only): query row r of batch b additionally does NOT see keys in [seg_lo, q_seg[b*Sq + r]).
  // Several continuations of one cached prefix (the answer options of vstar_bench_eval.py:127-163) are appended back to back
  // after the prefix and each row attends the prefix + the earlier rows of ITS OWN continuation only.
  const int* q_seg = nullptr;
  int seg_lo = 0;
};

constexpr int FA_BN = 64;

// swizzled element offset of (row, 16B-chunk) in a [rows][D] tile of a 2-byte type
template <int D>
__device__ __forceinline__ int swz(int row, int chunk) { return row * D + ((chunk ^ (row & 7)) << 3); }

template <int D, int ROWS, typename T>
__device__ __forceinline__ void load_tile(T* s, const T* g, long long rs, int row0, int nrows_valid, int tid) {
  constexpr int CH = D / 8;
  for (int i = tid; i < ROWS * CH; i += 128) {
    const int r = i / CH, c = i - r * CH;
    const bool ok = (row0 + r) < nrows_valid;
    const int rr = ok ? (row0 + r) : 0;
    cp_async16(s + swz<D>(r, c), g + (long long)rr * rs + c * 8, ok);
  }
}

// MT = m16 tiles per warp: a CTA (4 warps) owns BM = 64*MT query rows; each K/V fragment loaded from shared memory
// (ldmatrix) is reused by the MT row tiles of the warp, halving shared-memory traffic per flop at MT = 2.
template <int D, int MT, typename T>
__global__ void __launch_bounds__(128) flash_attn_kernel(const AttnParams p) {
  using E = ElemT<T>;
  constexpr int BM = 64 * MT;
  extern __shared__ __align__(128) uint8_t fa_smem[];
  T* sQ = reinterpret_cast<T*>(fa_smem);
  T* sK = sQ + BM * D;                  // [2][64][D]
  T* sV = sK + 2 * FA_BN * D;           // [2][64][D]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int m_blk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q0 = m_blk * BM;
  const T* qg = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_bs + (long long)h * D;
  const T* kg = reinterpret_cast<const T*>(p.k) + (long long)b * p.k_bs + (long long)h * D;
  const T* vg = reinterpret_cast<const T*>(p.v) + (long long)b * p.v_bs + (long long)h * D;
  const int off = p.Sk - p.Sq;

  int n_blocks = (p.Sk + FA_BN - 1) / FA_BN;
  if (p.causal) {
    int last_key = q0 + BM - 1 + off;               // largest key any query of this tile may see
    if (last_key > p.Sk - 1) last_key = p.Sk - 1;
    if (last_key < 0) last_key = 0;
    const int nb = last_key / FA_BN + 1;
    if (nb < n_blocks) n_blocks = nb;
  }

  load_tile<D, BM>(sQ, qg, p.q_rs, q0, p.Sq, tid);
  load_tile<D, FA_BN>(sK, kg, p.k_rs, 0, p.Sk, tid);
  load_tile<D, FA_BN>(sV, vg, p.v_rs, 0, p.Sk, tid);
  cp_async_commit();

  uint32_t qf[MT][D / 16][4];
  float o_acc[MT][D / 8][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < D / 8; ++i) { o_acc[mt][i][0] = o_acc[mt][i][1] = o_acc[mt][i][2] = o_acc[mt][i][3] = 0.f; }
  float row_max[MT][2], row_sum[MT][2];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { row_max[mt][0] = row_max[mt][1] = -INFINITY; row_sum[mt][0] = row_sum[mt][1] = 0.f; }
  const int wrow = warp * 16 * MT;      // this warp's first query row inside the CTA tile

  for (int nb = 0; nb < n_blocks; ++nb) {
    const int buf = nb & 1;
    cp_async_wait<0>();
    __syncthreads();
    if (nb + 1 < n_blocks) {
      load_tile<D, FA_BN>(sK + (buf ^ 1) * FA_BN * D, kg, p.k_rs, (nb + 1) * FA_BN, p.Sk, tid);
      load_tile<D, FA_BN>(sV + (buf ^ 1) * FA_BN * D, vg, p.v_rs, (nb + 1) * FA_BN, p.Sk, tid);
      cp_async_commit();
    }
    if (nb == 0) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk)
          ldmatrix_x4(qf[mt][kk][0], qf[mt][kk][1], qf[mt][kk][2], qf[mt][kk][3],
                      smem_u32(sQ + swz<D>(wrow + mt * 16 + (lane & 15), kk * 2 + (lane >> 4))));
    }
    const T* cK = sK + buf * FA_BN * D;
    const T* cV = sV + buf * FA_BN * D;

    // ---- S = Q K^T : (16*MT) x 64 per warp
    float s[MT][8][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[mt][i][0] = s[mt][i][1] = s[mt][i][2] = s[mt][i][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t r0, r1, r2, r3;
        ldmatrix_x4(r0, r1, r2, r3, smem_u32(cK + swz<D>(np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1))));
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma_16816<T>(s[mt][2 * np], qf[mt][kk], r0, r1);
          mma_16816<T>(s[mt][2 * np + 1], qf[mt][kk], r2, r3);
        }
      }
    }
    // ---- scale, mask, online softmax (rows g and g+8 of each 16-row tile)
    const int key0 = nb * FA_BN;
    uint32_t pf[MT][4][4];   // P as A-fragments for 4 k16 steps over the 64 keys
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const int qrow0 = q0 + wrow + mt * 16 + g;
      int seg[2] = {0, 0};
      if (p.q_seg) {
        seg[0] = (qrow0 < p.Sq) ? p.q_seg[(long long)b * p.Sq + qrow0] : 0;
        seg[1] = (qrow0 + 8 < p.Sq) ? p.q_seg[(long long)b * p.Sq + qrow0 + 8] : 0;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + i * 8 + 2 * t + (e & 1);
          const int qr = qrow0 + ((e >> 1) << 3);
          float x = s[mt][i][e] * p.scale_log2;
          const bool masked = (key >= p.Sk) || (p.causal && key > qr + off) || (key >= p.seg_lo && key < seg[e >> 1]);
          x = masked ? -INFINITY : x;
          s[mt][i][e] = x;
          mx[e >> 1] = fmaxf(mx[e >> 1], x);
        }
      }
      float corr[2], mnew[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float m = mx[r];
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        mnew[r] = fmaxf(row_max[mt][r], m);
        const float msafe = (mnew[r] == -INFINITY) ? 0.f : mnew[r];
        corr[r] = exp2f(row_max[mt][r] - msafe);     // row_max = -inf -> 0
        row_max[mt][r] = mnew[r];
        mnew[r] = msafe;
      }
      float psum[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float p0 = exp2f(s[mt][i][0] - mnew[0]);
        const float p1 = exp2f(s[mt][i][1] - mnew[0]);
        const float p2 = exp2f(s[mt][i][2] - mnew[1]);
        const float p3 = exp2f(s[mt][i][3] - mnew[1]);
        psum[0] += p0 + p1;
        psum[1] += p2 + p3;
        // the reference casts the softmax output to its dtype (bf16 / f16) before P@V
        pf[mt][i >> 1][(i & 1) * 2 + 0] = E::pack2(p0, p1);
        pf[mt][i >> 1][(i & 1) * 2 + 1] = E::pack2(p2, p3);
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) row_sum[mt][r] = row_sum[mt][r] * corr[r] + psum[r];
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o_acc[mt][i][0] *= corr[0]; o_acc[mt][i][1] *= corr[0];
        o_acc[mt][i][2] *= corr[1]; o_acc[mt][i][3] *= corr[1];
      }
    }
    // ---- O += P V
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int dp = 0; dp < D / 16; ++dp) {
        uint32_t r0, r1, r2, r3;
        ldmatrix_x4_trans(r0, r1, r2, r3, smem_u32(cV + swz<D>(ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), dp * 2 + (lane >> 4))));
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma_16816<T>(o_acc[mt][2 * dp], pf[mt][ks], r0, r1);
          mma_16816<T>(o_acc[mt][2 * dp + 1], pf[mt][ks], r2, r3);
        }
      }
    }
  }

  // ---- finalize: O /= row_sum, stage through smem (reuse sQ), coalesced 16 B stores
  __syncthreads();   // everyone is done reading sQ fragments / K / V
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float sum = row_sum[mt][r];
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      inv[r] = (sum > 0.f) ? 1.f / sum : 0.f;
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      const int r_lo = wrow + mt * 16 + g, r_hi = r_lo + 8;
      *reinterpret_cast<uint32_t*>(sQ + swz<D>(r_lo, i) + 2 * t) = E::pack2(o_acc[mt][i][0] * inv[0], o_acc[mt][i][1] * inv[0]);
      *reinterpret_cast<uint32_t*>(sQ + swz<D>(r_hi, i) + 2 * t) = E::pack2(o_acc[mt][i][2] * inv[1], o_acc[mt][i][3] * inv[1]);
    }
  }
  __syncthreads();
  T* og = reinterpret_cast<T*>(p.o) + (long long)b * p.o_bs + (long long)h * D;
  constexpr int CH = D / 8;
  for (int i = tid; i < BM * CH; i += 128) {
    const int r = i / CH, c = i - r * CH;
    if (q0 + r < p.Sq) *reinterpret_cast<uint4*>(og + (long long)(q0 + r) * p.o_rs + c * 8) = *reinterpret_cast<const uint4*>(sQ + swz<D>(r, c));
  }
}

// ------------------------------------------------------------------------------------------------
// small attention (SAM two-way transformer): one warp per (batch, head, query); keys strided over lanes.
// q [B, Nq, H*D], k/v [B, Nk, H*D] contiguous rows (row stride = ld*), D in {16, 32}.
template <int D, typename T>
__global__ void __launch_bounds__(128) attn_small_kernel(const T* __restrict__ q, long long ldq, const T* __restrict__ k,
                                                         long long ldk, const T* __restrict__ v, long long ldv,
                                                         T* __restrict__ o, long long ldo, int B, int H, int Nq, int Nk,
                                                         float scale) {
  using E = ElemT<T>;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = (long long)B * H * Nq;
  if (wid >= total) return;
  const int qi = wid % Nq;
  const int h = (wid / Nq) % H;
  const int b = wid / ((long long)Nq * H);
  const T* qp = q + ((long long)b * Nq + qi) * ldq + h * D;
  float qv[D];
#pragma unroll
  for (int d = 0; d < D; d += 2) {
    float2 f = E::unpack2(*reinterpret_cast<const uint32_t*>(qp + d));
    qv[d] = f.x * scale; qv[d + 1] = f.y * scale;
  }
  float m = -INFINITY, l = 0.f;
  float acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  for (int j = lane; j < Nk; j += 32) {
    const T* kp = k + ((long long)b * Nk + j) * ldk + h * D;
    const T* vp = v + ((long long)b * Nk + j) * ldv + h * D;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < D; d += 8) {
      uint4 u = *reinterpret_cast<const uint4*>(kp + d);
      float2 f;
      f = E::unpack2(u.x); s += qv[d] * f.x + qv[d + 1] * f.y;
      f = E::unpack2(u.y); s += qv[d + 2] * f.x + qv[d + 3] * f.y;
      f = E::unpack2(u.z); s += qv[d + 4] * f.x + qv[d + 5] * f.y;
      f = E::unpack2(u.w); s += qv[d + 6] * f.x + qv[d + 7] * f.y;
    }
    const float mn = fmaxf(m, s);
    const float c = __expf(m - mn);
    const float pj = __expf(s - mn);
    l = l * c + pj;
#pragma unroll
    for (int d = 0; d < D; d += 8) {
      uint4 u = *reinterpret_cast<const uint4*>(vp + d);
      float2 f;
      f = E::unpack2(u.x); acc[d] = acc[d] * c + pj * f.x; acc[d + 1] = acc[d + 1] * c + pj * f.y;
      f = E::unpack2(u.y); acc[d + 2] = acc[d + 2] * c + pj * f.x; acc[d + 3] = acc[d + 3] * c + pj * f.y;
      f = E::unpack2(u.z); acc[d + 4] = acc[d + 4] * c + pj * f.x; acc[d + 5] = acc[d + 5] * c + pj * f.y;
      f = E::unpack2(u.w); acc[d + 6] = acc[d + 6] * c + pj * f.x; acc[d + 7] = acc[d + 7] * c + pj * f.y;
    }
    m = mn;
  }
  // merge the 32 per-lane partial softmaxes
  float mg = warp_max(m);
  const float c = (m == -INFINITY) ? 0.f : __expf(m - mg);
  l = warp_sum(l * c);
  const float inv = 1.f / l;
  T* op = o + ((long long)b * Nq + qi) * ldo + h * D;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float a = warp_sum(acc[d] * c);
    if (lane == (d & 31)) op[d] = E::from_f(a * inv);   // (d & 31): spread the writers over the lanes
  }
}

}  // namespace

// wgmma kernel (attention_tc.cu)
template <typename T>
int vsb_flash_attn_tc(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs, long long k_rs,
                      long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, int D, int causal,
                      float scale, cudaStream_t stream);

// ------------------------------------------------------------------ decode attention (Sq <= 4 new rows against a long KV cache)
// HBM/latency-bound: one (batch, head) reads Sk rows of K and V once.  The FA2-style kernel above gives such a problem ONE
// CTA per head (32 CTAs for Vicuna-7B).  Here the keys of a head are split over a CLUSTER of 8
// CTAs (flash-decoding); each warp streams its keys with the row spread over the 32 lanes (coalesced 128/256 B rows, 4 keys
// in flight per warp), keeps an online-softmax partial (m, l, acc) per query, warps combine through shared memory, and
// cluster rank 0 combines the 8 CTA partials through DISTRIBUTED shared memory - no global scratch, no second kernel.
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

constexpr int DEC_SPLITS = 8;     // largest cluster size
constexpr int DEC_WARPS = 8;
constexpr int DEC_MAXQ = 4;
constexpr int DEC_U = 8;          // keys in flight per warp

template <int D, int NQ, typename T>      // NQ = compile-time bound on Sq (1 for plain decode, NQ otherwise)
__global__ void __launch_bounds__(DEC_WARPS * 32, 2) attn_decode_kernel(const AttnParams p) {
  using E = ElemT<T>;
  pdl_prologue();
  constexpr int EPL = D / 32;                                   // elements per lane
  cg::cluster_group cluster = cg::this_cluster();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float s_m[DEC_WARPS][NQ], s_l[DEC_WARPS][NQ];
  __shared__ float s_acc[DEC_WARPS][NQ][D];
  __shared__ float c_m[NQ], c_l[NQ];                // this CTA's combined partial (read remotely by rank 0)
  __shared__ float c_acc[NQ][D];

  const int off = p.Sk - p.Sq;
  const int k_first = p.k_start ? max(0, min(p.k_start[b], p.Sk)) : 0;
  const int nsplit = gridDim.x;                                 // = cluster size (1, 2, 4 or 8)
  const int chunk = (p.Sk - k_first + nsplit - 1) / nsplit;
  const int k_begin = k_first + split * chunk;
  const int k_end = min(p.Sk, k_begin + chunk);
  const T* qb = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_bs + (long long)h * D + lane * EPL;
  const T* kb = reinterpret_cast<const T*>(p.k) + (long long)b * p.k_bs + (long long)h * D + lane * EPL;
  const T* vb = reinterpret_cast<const T*>(p.v) + (long long)b * p.v_bs + (long long)h * D + lane * EPL;

  float q[NQ][EPL], acc[NQ][EPL], m[NQ], l[NQ];
#pragma unroll
  for (int qi = 0; qi < NQ; ++qi) {
    m[qi] = -INFINITY;
    l[qi] = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      acc[qi][e] = 0.f;
      q[qi][e] = (qi < p.Sq) ? E::to_f(qb[(long long)qi * p.q_rs + e]) * p.scale_log2 : 0.f;
    }
  }

  for (int j0 = k_begin + warp; j0 < k_end; j0 += DEC_WARPS * DEC_U) {
    // K / V rows stay packed (T pairs) until they are used: 2 x EPL/2 registers per key in flight
    uint32_t kr[DEC_U][EPL / 2], vr[DEC_U][EPL / 2];
#pragma unroll
    for (int u = 0; u < DEC_U; ++u) {
      const int j = j0 + u * DEC_WARPS;
      if (j < k_end) {
        if (EPL == 4) {
          const uint2 k2 = *reinterpret_cast<const uint2*>(kb + (long long)j * p.k_rs);
          const uint2 v2 = *reinterpret_cast<const uint2*>(vb + (long long)j * p.v_rs);
          kr[u][0] = k2.x; kr[u][(EPL / 2) - 1] = k2.y;
          vr[u][0] = v2.x; vr[u][(EPL / 2) - 1] = v2.y;
        } else {
          kr[u][0] = *reinterpret_cast<const uint32_t*>(kb + (long long)j * p.k_rs);
          vr[u][0] = *reinterpret_cast<const uint32_t*>(vb + (long long)j * p.v_rs);
        }
      } else {
#pragma unroll
        for (int e = 0; e < EPL / 2; ++e) kr[u][e] = vr[u][e] = 0u;
      }
    }
#pragma unroll
    for (int qi = 0; qi < NQ; ++qi) {
      if (qi < p.Sq) {                                          // warp-uniform
        const int jmax = p.causal ? qi + off : p.Sk - 1;
        float sc[DEC_U];
        float mx = m[qi];
#pragma unroll
        for (int u = 0; u < DEC_U; ++u) {
          float d = 0.f;
#pragma unroll
          for (int e = 0; e < EPL / 2; ++e) {
            const float2 kk = E::unpack2(kr[u][e]);
            d = fmaf(q[qi][2 * e], kk.x, d);
            d = fmaf(q[qi][2 * e + 1], kk.y, d);
          }
          d = warp_sum(d);
          const int j = j0 + u * DEC_WARPS;
          sc[u] = (j < k_end && j <= jmax) ? d : -INFINITY;
          mx = fmaxf(mx, sc[u]);
        }
        if (mx != -INFINITY) {
          const float corr = exp2f(m[qi] - mx);                 // m = -inf on first use -> 0
          m[qi] = mx;
          float ls = 0.f;
#pragma unroll
          for (int e = 0; e < EPL; ++e) acc[qi][e] *= corr;
#pragma unroll
          for (int u = 0; u < DEC_U; ++u) {
            const float pr = exp2f(sc[u] - mx);
            ls += pr;
#pragma unroll
            for (int e = 0; e < EPL / 2; ++e) {
              const float2 vv = E::unpack2(vr[u][e]);
              acc[qi][2 * e] = fmaf(pr, vv.x, acc[qi][2 * e]);
              acc[qi][2 * e + 1] = fmaf(pr, vv.y, acc[qi][2 * e + 1]);
            }
          }
          l[qi] = l[qi] * corr + ls;
        }
      }
    }
  }
  // warps -> CTA partial
#pragma unroll
  for (int qi = 0; qi < NQ; ++qi) {
    if (lane == 0) { s_m[warp][qi] = m[qi]; s_l[warp][qi] = l[qi]; }
#pragma unroll
    for (int e = 0; e < EPL; ++e) s_acc[warp][qi][lane * EPL + e] = acc[qi][e];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < NQ * D; idx += DEC_WARPS * 32) {
    const int qi = idx / D, d = idx - qi * D;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) M = fmaxf(M, s_m[w][qi]);
    float a = 0.f, ll = 0.f;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) {
      const float f = (s_m[w][qi] == -INFINITY) ? 0.f : exp2f(s_m[w][qi] - M);
      a += s_acc[w][qi][d] * f;
      ll += s_l[w][qi] * f;
    }
    c_acc[qi][d] = a;
    if (d == 0) { c_m[qi] = M; c_l[qi] = ll; }
  }
  cluster.sync();
  if (cluster.block_rank() == 0) {
    for (int idx = threadIdx.x; idx < p.Sq * D; idx += DEC_WARPS * 32) {
      const int qi = idx / D, d = idx - qi * D;
      float M = -INFINITY;
      for (int r = 0; r < nsplit; ++r) M = fmaxf(M, *cluster.map_shared_rank(&c_m[qi], r));
      float a = 0.f, ll = 0.f;
      for (int r = 0; r < nsplit; ++r) {
        const float mr = *cluster.map_shared_rank(&c_m[qi], r);
        const float f = (mr == -INFINITY) ? 0.f : exp2f(mr - M);
        a += *cluster.map_shared_rank(&c_acc[qi][d], r) * f;
        ll += *cluster.map_shared_rank(&c_l[qi], r) * f;
      }
      reinterpret_cast<T*>(p.o)[(long long)b * p.o_bs + (long long)qi * p.o_rs + (long long)h * D + d] = E::from_f(ll > 0.f ? a / ll : 0.f);
    }
  }
  cluster.sync();                                               // peers' shared memory must outlive rank 0's reads
}

template <int D, typename T>
static int launch_decode(const AttnParams& p, cudaStream_t st) {
  // keys of one (batch, head) are split over a cluster of 1..8 CTAs: as many as keep the machine filled about twice, but
  // not so many that a CTA gets fewer than ~64 keys (a batched decode step already has B*H independent heads)
  int splits = DEC_SPLITS;
  while (splits > 1 && ((long long)splits * p.H * p.B > 2LL * vsb_num_sms() + p.H || p.Sk / splits < 64)) splits >>= 1;
  if (p.Sq == 1)
    VSB_CUDA(vsb_launch_pdl(attn_decode_kernel<D, 1, T>, dim3(splits, p.H, p.B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  else
    VSB_CUDA(vsb_launch_pdl(attn_decode_kernel<D, DEC_MAXQ, T>, dim3(splits, p.H, p.B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  return VSB_OK;
}

// ------------------------------------------------------------------ decode attention over per-row cache slots and lengths
// A decode batch whose rows were admitted at different times: row b owns cache slot slot[b] and has len[b] cached rows; its
// query is the row the QKV step has just written, slot[b]*slot_stride + len[b]*row_stride, and it attends keys [0, len[b]] of
// its slot.  The kernel above with Sq = 1, except that the split of a row comes from its OWN key count: launch_decode's rule
// for Sk = len[b] + 1, with the batch-size term folded into `cap` on the host (dropped in batch-invariant mode, so a row's
// result depends on nothing but its own keys).  Surplus CTAs of the cluster stream no keys and rank 0 combines only the
// row's own splits, in rank order: in the default mode, with equal lengths and slot[b] = b, this is vsb_attn_decode_* with
// k_start = 0, bit for bit (in batch-invariant mode vsb_attn_decode_* keeps the batch-size term, so the splits may differ).
struct SlotAttnParams {
  const void *q, *k, *v;
  void* o;
  long long slot_stride, row_stride, o_rs;
  const int *slot, *len;
  float scale_log2;
  int cap;                       // largest split the batch-size term of launch_decode allows (1..8)
};

__device__ __forceinline__ int dec_row_splits(int nk, int cap) {
  int s = cap;
  while (s > 1 && nk / s < 64) s >>= 1;
  return s;
}

// the paged form (vsb_attn_decode_paged): row b's keys / values live in pages of 2^page_shift rows, key j at page
// page_table[slot[b]*pt_ld + (j >> page_shift)], row j & (page rows - 1); its query is row b of a separate q buffer (stride q_rs)
struct PagedSlotAttnParams {
  const void *q, *k, *v;
  void* o;
  long long page_stride, row_stride, o_rs, q_rs;
  const int *slot, *len, *page_table;
  float scale_log2;
  int cap;
  int pt_ld, page_shift;
};

// one body for both forms: only the addresses of q and of key row j differ, so a row's arithmetic (split rule, key chunks,
// combine order) is the same in both and they agree bit for bit on the same logical keys
template <int D, typename T, typename PRM>
__device__ __forceinline__ void attn_decode_slots_body(const PRM& p) {
  constexpr bool PAGED = std::is_same<PRM, PagedSlotAttnParams>::value;
  using E = ElemT<T>;
  pdl_prologue();
  constexpr int EPL = D / 32;
  cg::cluster_group cluster = cg::this_cluster();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float s_m[DEC_WARPS], s_l[DEC_WARPS];
  __shared__ float s_acc[DEC_WARPS][D];
  __shared__ float c_m, c_l;
  __shared__ float c_acc[D];

  const int len = p.len[b];
  const int nk = len + 1;
  const int nsplit = min(dec_row_splits(nk, p.cap), (int)gridDim.x);
  const int chunk = (nk + nsplit - 1) / nsplit;
  const int k_begin = split < nsplit ? split * chunk : nk;
  const int k_end = min(nk, k_begin + chunk);
  const T *qb, *kb, *vb;
  const int* pages = nullptr;
  if constexpr (PAGED) {
    const long long hoff = (long long)h * D + lane * EPL;
    qb = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_rs + hoff;
    kb = reinterpret_cast<const T*>(p.k) + hoff;
    vb = reinterpret_cast<const T*>(p.v) + hoff;
    pages = p.page_table + (long long)p.slot[b] * p.pt_ld;
  } else {
    const long long base = (long long)p.slot[b] * p.slot_stride + (long long)h * D + lane * EPL;
    qb = reinterpret_cast<const T*>(p.q) + base + (long long)len * p.row_stride;
    kb = reinterpret_cast<const T*>(p.k) + base;
    vb = reinterpret_cast<const T*>(p.v) + base;
  }
  // element offset of key / value row j from kb / vb
  auto row_off = [&](int j) -> long long {
    if constexpr (PAGED)
      return (long long)__ldg(pages + (j >> p.page_shift)) * p.page_stride + (long long)(j & ((1 << p.page_shift) - 1)) * p.row_stride;
    else
      return (long long)j * p.row_stride;
  };

  float q[EPL], acc[EPL], m = -INFINITY, l = 0.f;
#pragma unroll
  for (int e = 0; e < EPL; ++e) {
    acc[e] = 0.f;
    q[e] = E::to_f(qb[e]) * p.scale_log2;
  }
  for (int j0 = k_begin + warp; j0 < k_end; j0 += DEC_WARPS * DEC_U) {
    uint32_t kr[DEC_U][EPL / 2], vr[DEC_U][EPL / 2];
#pragma unroll
    for (int u = 0; u < DEC_U; ++u) {
      const int j = j0 + u * DEC_WARPS;
      if (j < k_end) {
        const long long ro = row_off(j);
        if (EPL == 4) {
          const uint2 k2 = *reinterpret_cast<const uint2*>(kb + ro);
          const uint2 v2 = *reinterpret_cast<const uint2*>(vb + ro);
          kr[u][0] = k2.x; kr[u][(EPL / 2) - 1] = k2.y;
          vr[u][0] = v2.x; vr[u][(EPL / 2) - 1] = v2.y;
        } else {
          kr[u][0] = *reinterpret_cast<const uint32_t*>(kb + ro);
          vr[u][0] = *reinterpret_cast<const uint32_t*>(vb + ro);
        }
      } else {
#pragma unroll
        for (int e = 0; e < EPL / 2; ++e) kr[u][e] = vr[u][e] = 0u;
      }
    }
    float sc[DEC_U];
    float mx = m;
#pragma unroll
    for (int u = 0; u < DEC_U; ++u) {
      float d = 0.f;
#pragma unroll
      for (int e = 0; e < EPL / 2; ++e) {
        const float2 kk = E::unpack2(kr[u][e]);
        d = fmaf(q[2 * e], kk.x, d);
        d = fmaf(q[2 * e + 1], kk.y, d);
      }
      d = warp_sum(d);
      sc[u] = (j0 + u * DEC_WARPS < k_end) ? d : -INFINITY;
      mx = fmaxf(mx, sc[u]);
    }
    if (mx != -INFINITY) {
      const float corr = exp2f(m - mx);
      m = mx;
      float ls = 0.f;
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[e] *= corr;
#pragma unroll
      for (int u = 0; u < DEC_U; ++u) {
        const float pr = exp2f(sc[u] - mx);
        ls += pr;
#pragma unroll
        for (int e = 0; e < EPL / 2; ++e) {
          const float2 vv = E::unpack2(vr[u][e]);
          acc[2 * e] = fmaf(pr, vv.x, acc[2 * e]);
          acc[2 * e + 1] = fmaf(pr, vv.y, acc[2 * e + 1]);
        }
      }
      l = l * corr + ls;
    }
  }
  // warps -> CTA partial -> rank 0, in the order of attn_decode_kernel
  if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
#pragma unroll
  for (int e = 0; e < EPL; ++e) s_acc[warp][lane * EPL + e] = acc[e];
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += DEC_WARPS * 32) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) M = fmaxf(M, s_m[w]);
    float a = 0.f, ll = 0.f;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) {
      const float f = (s_m[w] == -INFINITY) ? 0.f : exp2f(s_m[w] - M);
      a += s_acc[w][d] * f;
      ll += s_l[w] * f;
    }
    c_acc[d] = a;
    if (d == 0) { c_m = M; c_l = ll; }
  }
  cluster.sync();
  if (cluster.block_rank() == 0) {
    for (int d = threadIdx.x; d < D; d += DEC_WARPS * 32) {
      float M = -INFINITY;
      for (int r = 0; r < nsplit; ++r) M = fmaxf(M, *cluster.map_shared_rank(&c_m, r));
      float a = 0.f, ll = 0.f;
      for (int r = 0; r < nsplit; ++r) {
        const float mr = *cluster.map_shared_rank(&c_m, r);
        const float f = (mr == -INFINITY) ? 0.f : exp2f(mr - M);
        a += *cluster.map_shared_rank(&c_acc[d], r) * f;
        ll += *cluster.map_shared_rank(&c_l, r) * f;
      }
      reinterpret_cast<T*>(p.o)[(long long)b * p.o_rs + (long long)h * D + d] = E::from_f(ll > 0.f ? a / ll : 0.f);
    }
  }
  cluster.sync();
}

template <int D, typename T>
__global__ void __launch_bounds__(DEC_WARPS * 32, 2) attn_decode_slots_kernel(const SlotAttnParams p) {
  attn_decode_slots_body<D, T>(p);
}

template <int D, typename T>
__global__ void __launch_bounds__(DEC_WARPS * 32, 2) attn_decode_paged_kernel(const PagedSlotAttnParams p) {
  attn_decode_slots_body<D, T>(p);
}

// launch_decode's rule, split into its batch-size term (the returned cap) and its key-count term (per row in the kernel; here
// for the longest row, which sizes the cluster: *splits)
static int slot_split_cap(int B, int H, int max_len, int* splits) {
  int cap = DEC_SPLITS;
  if (!vsb_batch_invariant())
    while (cap > 1 && (long long)cap * H * B > 2LL * vsb_num_sms() + H) cap >>= 1;
  int s = cap;
  while (s > 1 && (max_len + 1) / s < 64) s >>= 1;
  *splits = s;
  return cap;
}

template <typename T>
static int attn_decode_slots(const void* q, const void* k, const void* v, void* o, long long slot_stride, long long row_stride, long long o_rs,
                             int B, int H, int D, float scale, const void* slot, const void* len, int max_len, void* stream) {
  VSB_CHECK_ARG(q && k && v && o && slot && len, "vsb_attn_decode_slots: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_attn_decode_slots: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(B > 0 && H > 0 && max_len >= 0, "vsb_attn_decode_slots: bad shape (B=%d, H=%d, max_len=%d)", B, H, max_len);
  VSB_CHECK_ARG(slot_stride % 4 == 0 && row_stride % 4 == 0 && ((uintptr_t)q & 7) == 0 && ((uintptr_t)k & 7) == 0 && ((uintptr_t)v & 7) == 0,
                "vsb_attn_decode_slots: q/k/v must be 8-byte aligned with strides that are multiples of 4 elements");
  SlotAttnParams p;
  p.q = q; p.k = k; p.v = v; p.o = o;
  p.slot_stride = slot_stride; p.row_stride = row_stride; p.o_rs = o_rs;
  p.slot = reinterpret_cast<const int*>(slot); p.len = reinterpret_cast<const int*>(len);
  p.scale_log2 = scale * 1.4426950408889634f;
  int splits;
  p.cap = slot_split_cap(B, H, max_len, &splits);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D == 64)
    VSB_CUDA(vsb_launch_pdl(attn_decode_slots_kernel<64, T>, dim3(splits, H, B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  else
    VSB_CUDA(vsb_launch_pdl(attn_decode_slots_kernel<128, T>, dim3(splits, H, B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  return VSB_OK;
}

template <typename T>
static int attn_decode_paged(const void* q, long long q_rs, const void* k, const void* v, void* o, long long o_rs, long long page_stride,
                             long long row_stride, int page_rows, const void* page_table, int pt_ld, int B, int H, int D, float scale,
                             const void* slot, const void* len, int max_len, void* stream) {
  VSB_CHECK_ARG(q && k && v && o && page_table && slot && len, "vsb_attn_decode_paged: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_attn_decode_paged: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(B > 0 && H > 0 && max_len >= 0 && pt_ld > 0, "vsb_attn_decode_paged: bad shape (B=%d, H=%d, max_len=%d, pt_ld=%d)", B, H,
                max_len, pt_ld);
  VSB_CHECK_ARG(page_rows >= 16 && (page_rows & (page_rows - 1)) == 0, "vsb_attn_decode_paged: page_rows %d is not a power of two >= 16",
                page_rows);
  VSB_CHECK_ARG((long long)max_len < (long long)pt_ld * page_rows, "vsb_attn_decode_paged: max_len %d past the %d x %d rows of a page table row",
                max_len, pt_ld, page_rows);
  VSB_CHECK_ARG(q_rs % 4 == 0 && page_stride % 4 == 0 && row_stride % 4 == 0 && ((uintptr_t)q & 7) == 0 && ((uintptr_t)k & 7) == 0 &&
                    ((uintptr_t)v & 7) == 0,
                "vsb_attn_decode_paged: q/k/v must be 8-byte aligned with strides that are multiples of 4 elements");
  PagedSlotAttnParams p;
  p.q = q; p.k = k; p.v = v; p.o = o;
  p.page_stride = page_stride; p.row_stride = row_stride; p.o_rs = o_rs; p.q_rs = q_rs;
  p.slot = reinterpret_cast<const int*>(slot); p.len = reinterpret_cast<const int*>(len);
  p.page_table = reinterpret_cast<const int*>(page_table);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.pt_ld = pt_ld;
  p.page_shift = __builtin_ctz((unsigned)page_rows);
  int splits;
  p.cap = slot_split_cap(B, H, max_len, &splits);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D == 64)
    VSB_CUDA(vsb_launch_pdl(attn_decode_paged_kernel<64, T>, dim3(splits, H, B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  else
    VSB_CUDA(vsb_launch_pdl(attn_decode_paged_kernel<128, T>, dim3(splits, H, B), dim3(DEC_WARPS * 32), 0, st, splits, p));
  return VSB_OK;
}

void vsb_attn_tc_set_variant(int v);
static int g_attn_impl = 0;   // 0 auto, 1 = mma.sync kernel, 2 = wgmma kernel, 3 = wgmma kernel with one query warpgroup per CTA, 4 = decode kernel
extern "C" int vsb_attn_set_impl(int impl) {
  g_attn_impl = (impl == 3) ? 2 : impl;
  vsb_attn_tc_set_variant(impl == 3 ? 1 : 0);
  return VSB_OK;
}

template <typename T>
static int attn_decode(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs,
                                    long long k_bs, long long k_rs, long long v_bs, long long v_rs, long long o_bs,
                                    long long o_rs, int B, int H, int Sq, int Sk, int D, int causal, float scale,
                                    const void* k_start, void* stream) {
  VSB_CHECK_ARG(q && k && v && o, "vsb_attn_decode_bf16: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_attn_decode_bf16: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Sk > 0 && Sq <= DEC_MAXQ, "vsb_attn_decode_bf16: bad shape (Sq=%d, at most %d)", Sq, DEC_MAXQ);
  VSB_CHECK_ARG(q_rs % 4 == 0 && k_rs % 4 == 0 && v_rs % 4 == 0 && q_bs % 4 == 0 && k_bs % 4 == 0 && v_bs % 4 == 0 &&
                    ((uintptr_t)q & 7) == 0 && ((uintptr_t)k & 7) == 0 && ((uintptr_t)v & 7) == 0,
                "vsb_attn_decode_bf16: q/k/v must be 8-byte aligned with strides that are multiples of 4 elements");
  AttnParams pd;
  pd.q = q; pd.k = k; pd.v = v; pd.o = o;
  pd.q_bs = q_bs; pd.q_rs = q_rs; pd.k_bs = k_bs; pd.k_rs = k_rs; pd.v_bs = v_bs; pd.v_rs = v_rs; pd.o_bs = o_bs; pd.o_rs = o_rs;
  pd.B = B; pd.H = H; pd.Sq = Sq; pd.Sk = Sk; pd.causal = causal;
  pd.scale_log2 = scale * 1.4426950408889634f;
  pd.k_start = reinterpret_cast<const int*>(k_start);
  return D == 64 ? launch_decode<64, T>(pd, reinterpret_cast<cudaStream_t>(stream)) : launch_decode<128, T>(pd, reinterpret_cast<cudaStream_t>(stream));
}

template <typename T>
static int launch_flash_mma(const AttnParams& p, int D, cudaStream_t st) {
  if (D == 64) {
    const int smem = (64 + 4 * FA_BN) * 64 * 2;
    static bool set64 = false;
    if (!set64) { VSB_CUDA(cudaFuncSetAttribute(flash_attn_kernel<64, 1, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); set64 = true; }
    dim3 grid((p.Sq + 63) / 64, p.H, p.B);
    flash_attn_kernel<64, 1, T><<<grid, 128, smem, st>>>(p);
  } else {
    const int smem = (64 + 4 * FA_BN) * 128 * 2;
    static bool set128 = false;
    if (!set128) { VSB_CUDA(cudaFuncSetAttribute(flash_attn_kernel<128, 1, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); set128 = true; }
    dim3 grid((p.Sq + 63) / 64, p.H, p.B);
    flash_attn_kernel<128, 1, T><<<grid, 128, smem, st>>>(p);
  }
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename T>
static int flash_attn(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs,
                                   long long k_bs, long long k_rs, long long v_bs, long long v_rs, long long o_bs,
                                   long long o_rs, int B, int H, int Sq, int Sk, int D, int causal, float scale, void* stream) {
  VSB_CHECK_ARG(q && k && v && o, "vsb_flash_attn_bf16: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_flash_attn_bf16: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Sk > 0, "vsb_flash_attn_bf16: bad shape");
  VSB_CHECK_ARG(q_rs % 8 == 0 && k_rs % 8 == 0 && v_rs % 8 == 0 && o_rs % 8 == 0 && q_bs % 8 == 0 && k_bs % 8 == 0 &&
                    v_bs % 8 == 0 && o_bs % 8 == 0,
                "vsb_flash_attn_bf16: strides must be multiples of 8 elements (16 B)");
  VSB_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0 && ((uintptr_t)o & 15) == 0,
                "vsb_flash_attn_bf16: pointers must be 16-byte aligned");
  if (g_attn_impl == 4 || (g_attn_impl == 0 && Sq <= DEC_MAXQ && Sk >= 64))
    return attn_decode<T>(q, k, v, o, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs, B, H, Sq, Sk, D, causal, scale, nullptr, stream);
  if (g_attn_impl == 2 || (g_attn_impl == 0 && Sq >= 64))
    return vsb_flash_attn_tc<T>(q, k, v, o, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs, B, H, Sq, Sk, D, causal, scale,
                             reinterpret_cast<cudaStream_t>(stream));
  AttnParams p;
  p.q = q; p.k = k; p.v = v; p.o = o;
  p.q_bs = q_bs; p.q_rs = q_rs; p.k_bs = k_bs; p.k_rs = k_rs; p.v_bs = v_bs; p.v_rs = v_rs; p.o_bs = o_bs; p.o_rs = o_rs;
  p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  return launch_flash_mma<T>(p, D, reinterpret_cast<cudaStream_t>(stream));
}

// Causal attention of several CONTINUATIONS of one cached prefix in one launch (answer-option scoring of the SEAL VQA LLM,
// /root/reference/vstar_bench_eval.py:127-163, where the reference runs one forward per option on the question's
// past_key_values): the Sq new rows sit at keys Sk-Sq .. Sk-1; row r sees keys 0..seg_lo-1 (the prefix) and
// q_seg[b*Sq + r] .. (Sk-Sq+r) (the earlier rows of its own continuation).  mma.sync kernel (Sq is a few dozen rows).
template <typename T>
static int flash_attn_seg(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs,
                                       long long k_bs, long long k_rs, long long v_bs, long long v_rs, long long o_bs,
                                       long long o_rs, int B, int H, int Sq, int Sk, int D, float scale, const void* q_seg_i32, int seg_lo,
                                       void* stream) {
  VSB_CHECK_ARG(q && k && v && o && q_seg_i32, "vsb_flash_attn_seg_bf16: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_flash_attn_seg_bf16: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Sk >= Sq && seg_lo >= 0 && seg_lo <= Sk, "vsb_flash_attn_seg_bf16: bad shape");
  VSB_CHECK_ARG(q_rs % 8 == 0 && k_rs % 8 == 0 && v_rs % 8 == 0 && o_rs % 8 == 0 && q_bs % 8 == 0 && k_bs % 8 == 0 &&
                    v_bs % 8 == 0 && o_bs % 8 == 0,
                "vsb_flash_attn_seg_bf16: strides must be multiples of 8 elements (16 B)");
  AttnParams p;
  p.q = q; p.k = k; p.v = v; p.o = o;
  p.q_bs = q_bs; p.q_rs = q_rs; p.k_bs = k_bs; p.k_rs = k_rs; p.v_bs = v_bs; p.v_rs = v_rs; p.o_bs = o_bs; p.o_rs = o_rs;
  p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk; p.causal = 1;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.q_seg = reinterpret_cast<const int*>(q_seg_i32);
  p.seg_lo = seg_lo;
  return launch_flash_mma<T>(p, D, reinterpret_cast<cudaStream_t>(stream));
}

template <typename T>
static int attn_small(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o,
                                   long long ldo, int B, int H, int Nq, int Nk, int D, float scale, void* stream) {
  VSB_CHECK_ARG(q && k && v && o, "vsb_attn_small_bf16: null pointer");
  VSB_CHECK_ARG(D == 16 || D == 32 || D == 96, "vsb_attn_small_bf16: head_dim %d unsupported (16/32/96)", D);
  VSB_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0, "vsb_attn_small_bf16: ld must be multiples of 8");
  const long long warps = (long long)B * H * Nq;
  if (warps <= 0) return VSB_OK;
  const int blocks = (int)((warps + 3) / 4);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if constexpr (ElemT<T>::is_f16) {
    attn_small_kernel<96, T><<<blocks, 128, 0, st>>>((const T*)q, ldq, (const T*)k, ldk, (const T*)v, ldv, (T*)o, ldo, B, H, Nq, Nk, scale);
  } else if (D == 16)
    attn_small_kernel<16, T><<<blocks, 128, 0, st>>>((const T*)q, ldq, (const T*)k, ldk, (const T*)v, ldv, (T*)o, ldo, B, H, Nq, Nk, scale);
  else if (D == 32)
    attn_small_kernel<32, T><<<blocks, 128, 0, st>>>((const T*)q, ldq, (const T*)k, ldk, (const T*)v, ldv, (T*)o, ldo, B, H, Nq, Nk, scale);
  else   // SEAL perceiver resampler: 16 heads x 96, 32 latents <-> 288 keys (LLaVA/llava/model/multimodal_projector/perceiver.py:25-77)
    attn_small_kernel<96, T><<<blocks, 128, 0, st>>>((const T*)q, ldq, (const T*)k, ldk, (const T*)v, ldv, (T*)o, ldo, B, H, Nq, Nk, scale);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

// ------------------------------------------------------------------ C entry points: bf16 (VSM, default VQA engine) and f16 (VQA engine in fp16)
#define VSB_ATTN_ENTRY(NAME, IMPL, T)                                                                                              \
  extern "C" int NAME(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,        \
                      long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, \
                      int D, int causal, float scale, void* stream) {                                                                \
    return IMPL<T>(q, k, v, o, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs, B, H, Sq, Sk, D, causal, scale, stream);           \
  }
VSB_ATTN_ENTRY(vsb_flash_attn_bf16, flash_attn, bf16)
VSB_ATTN_ENTRY(vsb_flash_attn_f16, flash_attn, half)

#define VSB_ATTN_DECODE_ENTRY(NAME, T)                                                                                             \
  extern "C" int NAME(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,        \
                      long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, \
                      int D, int causal, float scale, const void* k_start, void* stream) {                                           \
    return attn_decode<T>(q, k, v, o, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs, B, H, Sq, Sk, D, causal, scale, k_start, stream); \
  }
VSB_ATTN_DECODE_ENTRY(vsb_attn_decode_bf16, bf16)
VSB_ATTN_DECODE_ENTRY(vsb_attn_decode_f16, half)

extern "C" int vsb_attn_decode_slots(const void* q, const void* k, const void* v, void* o, long long slot_stride, long long row_stride,
                                     long long o_rs, int B, int H, int D, float scale, const void* slot_i32, const void* len_i32, int max_len,
                                     int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_attn_decode_slots: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  return dtype == VSB_DTYPE_F16 ? attn_decode_slots<half>(q, k, v, o, slot_stride, row_stride, o_rs, B, H, D, scale, slot_i32, len_i32, max_len, stream)
                                : attn_decode_slots<bf16>(q, k, v, o, slot_stride, row_stride, o_rs, B, H, D, scale, slot_i32, len_i32, max_len, stream);
}

extern "C" int vsb_attn_decode_paged(const void* q, long long q_rs, const void* k, const void* v, void* o, long long o_rs, long long page_stride,
                                     long long row_stride, int page_rows, const void* page_table_i32, int pt_ld, int B, int H, int D, float scale,
                                     const void* slot_i32, const void* len_i32, int max_len, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_attn_decode_paged: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  return dtype == VSB_DTYPE_F16 ? attn_decode_paged<half>(q, q_rs, k, v, o, o_rs, page_stride, row_stride, page_rows, page_table_i32, pt_ld, B, H, D,
                                                          scale, slot_i32, len_i32, max_len, stream)
                                : attn_decode_paged<bf16>(q, q_rs, k, v, o, o_rs, page_stride, row_stride, page_rows, page_table_i32, pt_ld, B, H, D,
                                                          scale, slot_i32, len_i32, max_len, stream);
}

#define VSB_ATTN_SEG_ENTRY(NAME, T)                                                                                                \
  extern "C" int NAME(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,        \
                      long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, \
                      int D, float scale, const void* q_seg_i32, int seg_lo, void* stream) {                                         \
    return flash_attn_seg<T>(q, k, v, o, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs, B, H, Sq, Sk, D, scale, q_seg_i32, seg_lo, stream); \
  }
VSB_ATTN_SEG_ENTRY(vsb_flash_attn_seg_bf16, bf16)
VSB_ATTN_SEG_ENTRY(vsb_flash_attn_seg_f16, half)

extern "C" int vsb_attn_small_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o,
                                   long long ldo, int B, int H, int Nq, int Nk, int D, float scale, void* stream) {
  return attn_small<bf16>(q, ldq, k, ldk, v, ldv, o, ldo, B, H, Nq, Nk, D, scale, stream);
}
// f16: the perceiver resampler's head_dim 96 only (the SAM heads of 16 / 32 are bf16-only, like the rest of the VSM)
extern "C" int vsb_attn_small_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o,
                                  long long ldo, int B, int H, int Nq, int Nk, int D, float scale, void* stream) {
  VSB_CHECK_ARG(D == 96, "vsb_attn_small_f16: head_dim %d unsupported (96)", D);
  return attn_small<half>(q, ldq, k, ldk, v, ldv, o, ldo, B, H, Nq, Nk, D, scale, stream);
}
