// wgmma flash attention (prefill shapes): softmax(Q K^T * scale [+ causal]) V, head_dim 64 / 128, bf16 or f16, fp32 softmax.
//
// One CTA = NWG consumer warpgroups x 64 query rows of one (batch, head) + one producer warpgroup; keys are consumed in
// blocks of 128 that all consumer warpgroups share:
//   S  = Q K_j^T          wgmma m64n128k16 x D/16   (A = Q tile, B = K tile, both K-major SW128 from TMA) -> registers
//   P  = exp2(S*s - m)    on the accumulator fragments: a row lives in the 4 threads of a quad (max / sum by 2 shuffles)
//   O += P V_j            wgmma m64nDk16 x 8         (A = P straight from registers as T fragments, B = V tile as an
//                                                     MN-major operand: V stays [key][d]) -> O accumulates in registers
// The online-softmax rescale is lazy: the exponent reference m_ref of a row only moves when its running max grows by more
// than 2^8 (then O and l of that row are scaled by 2^(m_old - m_new)).
// Warpgroup 0: one thread issues the TMA loads (Q once, K/V ring via 3-D tensor maps so rows >= Sk are zero-filled).
//
// Replaces the mma.sync kernel of attention.cu for Sq >= 64 (CLIP S=257, OWL-ViT S=2305, 7B prefill T~320); numerics as
// the reference: scores and softmax in fp32, P rounded to T before P@V (modeling_clip.py:261-329, modeling_llama.py:199-221).
#include "common.cuh"
#include "vstar_b200.h"
#include "wgmma.cuh"

#include <mutex>
#include <type_traits>

namespace {

constexpr int BKV = 128;    // keys per block
constexpr int SUB_BYTES = 128 * 64 * 2;   // one [128][64] bf16 SW128 K / V sub-tile

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) { asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory"); }

// K-major SW128 operand (A = Q tile, B = K tile): SBO = 1024 B between 8-row groups (see gemm_tcgen05.cu)
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// MN-major SW128 operand (B = V tile kept as [key][d]): canonical layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units:
// 64 contiguous MN (= d) elements per 128-byte row, 8 consecutive K (= key) rows per 1024-byte swizzle atom,
// SBO = 1024 B between 8-key groups, LBO = stride between 64-wide d blocks (one 16 KB sub-tile)
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(SUB_BYTES >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// one MUFU op: 2^x, |rel err| <= 2^-22, ex2(-inf) = 0
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

struct AttnTcParams {
  void* o;
  long long o_bs, o_rs;
  int H, Sq, Sk, causal;
  float scale_log2;
};

template <int D, int NWG>
struct ASmem {
  static constexpr int NSUB = D / 64;
  static constexpr int KV_ST = (D == 64) ? 3 : 2;
  static constexpr int Q_SUB = NWG * 64 * 128;                     // one [64 NWG][64] bf16 SW128 Q sub-tile
  static constexpr int Q_BYTES = NSUB * Q_SUB;
  static constexpr int KV_STAGE_BYTES = 2 * NSUB * SUB_BYTES;      // K sub-tiles then V sub-tiles
  static constexpr int BAR_OFF = Q_BYTES + KV_ST * KV_STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 128;
};

// the paged chunk form (vsb_attn_chunk_paged): S segments of query rows, segment s = rows [lo, lo + n) of the request on
// page-table row slot, its queries rows [qoff, qoff + n) of q; key j of that request is row j % page_rows of page
// page_table[slot*pt_ld + j / page_rows], found in ONE tensor map over the pool's k|v rows from pool row `row0` (the layer) on
struct ChunkAttnParams {
  void* o;
  long long o_rs;
  const int* seg;          // int32 [3][S]: slot, lo, n
  const int* page_table;
  int S, H, pt_ld, page_rows, row0, d;
  float scale_log2;
};

// one body for both forms: only where the query tile's rows and the K/V tiles come from differ (and the paged form zeroes the V
// rows past the tile's last key, which a page may hold unwritten), so a row's scores, online softmax and P V are the same
// arithmetic in both, and fully masked key blocks add exact zeros: the forms agree bit for bit on the same logical keys
template <int D, int NWG, typename T, typename PRM>
__device__ __forceinline__ void attn_wgmma_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const PRM& p) {
  constexpr bool PAGED = std::is_same<PRM, ChunkAttnParams>::value;
  using L = ASmem<D, NWG>;
  constexpr int NSUB = L::NSUB;
  constexpr int ST = L::KV_ST;
  constexpr int BQ = 64 * NWG;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + L::Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;                 // [ST]
  uint64_t* kv_empty = kv_full + ST;            // [ST]

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  int q0, h, b, off, nblk;
  int lo = 0, n = 0, kend = 0, qoff = 0;
  const int* pages = nullptr;
  if constexpr (PAGED) {
    // tile blockIdx.x of the segments' tiles of BQ rows (a tile never spans two segments); CTAs past the last tile exit
    int tile = blockIdx.x, s = 0;
    for (; s < p.S; ++s) {
      n = p.seg[2 * p.S + s];
      const int nt = (n + BQ - 1) / BQ;
      if (tile < nt) break;
      tile -= nt;
      qoff += n;
    }
    if (s == p.S) return;
    lo = p.seg[p.S + s];
    pages = p.page_table + (long long)p.seg[s] * p.pt_ld;
    q0 = tile * BQ;                                    // segment-local first row of the tile
    h = blockIdx.y;
    b = 0;
    off = lo;                                          // row i attends keys [0, lo + i]
    kend = lo + min(q0 + BQ, n);                       // keys [0, kend) are written; the rows past it may hold anything
    nblk = (kend - 1) / BKV + 1;
  } else {
    q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
    off = p.Sk - p.Sq;
    nblk = (p.Sk + BKV - 1) / BKV;
    if (p.causal) {
      int last_key = q0 + BQ - 1 + off;
      if (last_key > p.Sk - 1) last_key = p.Sk - 1;
      if (last_key < 0) last_key = 0;
      const int nb = last_key / BKV + 1;
      if (nb < nblk) nblk = nb;
    }
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 4 * NWG); }   // one arrive per consumer warp
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ---------------- TMA producer
    if constexpr (NWG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, L::Q_BYTES);
#pragma unroll
      for (int s = 0; s < NSUB; ++s) tma_load_3d(sQ + s * L::Q_SUB, &tmQ, h * D + s * 64, PAGED ? qoff + q0 : q0, b, q_full);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nblk; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        uint8_t* dst = sKV + stage * L::KV_STAGE_BYTES;
        if constexpr (PAGED) {
          // a block of 128 keys is two boxes of 64 rows, each inside one page (page_rows % 64 == 0); a box wholly past the
          // tile's last key is not loaded (the consumers zero its V rows)
          const int halves = min(2, (kend - j * BKV + 63) / 64);
          mbar_arrive_expect_tx(&kv_full[stage], halves * (L::KV_STAGE_BYTES / 2));
          for (int hf = 0; hf < halves; ++hf) {
            const int key = j * BKV + hf * 64;
            const int row = p.row0 + __ldg(pages + key / p.page_rows) * p.page_rows + key % p.page_rows;
#pragma unroll
            for (int s = 0; s < NSUB; ++s) {
              tma_load_3d(dst + s * SUB_BYTES + hf * (SUB_BYTES / 2), &tmK, h * D + s * 64, row, 0, &kv_full[stage]);
              tma_load_3d(dst + (NSUB + s) * SUB_BYTES + hf * (SUB_BYTES / 2), &tmV, p.d + h * D + s * 64, row, 0, &kv_full[stage]);
            }
          }
        } else {
          mbar_arrive_expect_tx(&kv_full[stage], L::KV_STAGE_BYTES);
#pragma unroll
          for (int s = 0; s < NSUB; ++s) {
            tma_load_3d(dst + s * SUB_BYTES, &tmK, h * D + s * 64, j * BKV, b, &kv_full[stage]);
            tma_load_3d(dst + (NSUB + s) * SUB_BYTES, &tmV, h * D + s * 64, j * BKV, b, &kv_full[stage]);
          }
        }
        if (++stage == ST) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ---------------- consumers: warpgroup c owns query rows [64c, 64c + 64) of the CTA; thread rows r0 = 16 w + lane/4 and
  // r0 + 8, key / d columns 8 j + 2 t + {0, 1} of every fragment block j (t = lane % 4)
  if constexpr (NWG == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int c = wg - 1;
  const int t = lane & 3;
  const int rr = c * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int qrow[2] = {q0 + rr, q0 + rr + 8};
  int kmax[2];
  if constexpr (PAGED) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) kmax[hh] = min(qrow[hh] + off, kend - 1);
  } else {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) kmax[hh] = p.causal ? min(qrow[hh] + off, p.Sk - 1) : (p.Sk - 1);   // last visible key of the row
  }
  float m_ref[2] = {0.f, 0.f}, l_part[2] = {0.f, 0.f};
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float s[BKV / 2];
  const uint32_t aQ = smem_u32(sQ) + c * (64 * 128);

  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < nblk; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t aK = smem_u32(sKV + stage * L::KV_STAGE_BYTES);
    const uint32_t aV = aK + NSUB * SUB_BYTES;
    if constexpr (PAGED) {
      // V rows [kend - j*BKV, BKV) of the last block: unwritten page rows (or not loaded) -> zero, so P = 0 there adds exact zeros.
      // A SW128 row of a sub-tile is its 128 bytes whatever the swizzle; every consumer thread zeroes a share, then all of them
      // meet before any reads V
      const int z0 = kend - j * BKV;
      if (z0 < BKV) {
        uint8_t* sv = sKV + stage * L::KV_STAGE_BYTES + NSUB * SUB_BYTES;
        const int per_sub = (BKV - z0) * 8;             // 16-byte chunks per sub-tile
        for (int i = threadIdx.x - 128; i < NSUB * per_sub; i += 128 * NWG) {
          const int s = i / per_sub, r = i - s * per_sub;
          *reinterpret_cast<uint4*>(sv + s * SUB_BYTES + z0 * 128 + r * 16) = make_uint4(0, 0, 0, 0);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync 1, %0;" ::"r"(128 * NWG) : "memory");
      }
    }
    // ---- S = Q K_j^T
    fence_regs<BKV / 2>(s);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss<BKV, T>(s, desc_kmajor(aQ + (kk >> 2) * L::Q_SUB + (kk & 3) * 32), desc_kmajor(aK + (kk >> 2) * SUB_BYTES + (kk & 3) * 32),
                    kk > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<BKV / 2>(s);
    // ---- mask, row max (quad), lazy reference-max update
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int nvis = kmax[hh] - j * BKV + 1;        // keys [0, nvis) of the block are visible to this row
      if (nvis < BKV) {
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * jj + 2 * t + e >= nvis) s[4 * jj + 2 * hh + e] = -INFINITY;
      }
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) mx[hh] = fmaxf(mx[hh], fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      mx[hh] *= p.scale_log2;                          // scale > 0: max commutes with the scaling
      if (j == 0) {
        m_ref[hh] = (mx[hh] == -INFINITY) ? 0.f : mx[hh];
      } else if (mx[hh] > m_ref[hh] + 8.f) {
        const float corr = exp2f(m_ref[hh] - mx[hh]);
        m_ref[hh] = mx[hh];
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) { o[4 * jj + 2 * hh] *= corr; o[4 * jj + 2 * hh + 1] *= corr; }
        l_part[hh] *= corr;
      }
    }
    // ---- P = exp2(s * scale - m_ref) (<= 2^8) as T A fragments: block kk of 16 keys = accumulator blocks 2kk, 2kk+1
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {                  // q: (block 2kk + q/2, row q%2)
        const int hh = q & 1, base = 4 * (2 * kk + (q >> 1)) + 2 * hh;
        const float p0 = ex2_approx(fmaf(s[base], p.scale_log2, -m_ref[hh]));
        const float p1 = ex2_approx(fmaf(s[base + 1], p.scale_log2, -m_ref[hh]));
        l_part[hh] += p0 + p1;
        pa[kk][q] = ElemT<T>::pack2(p0, p1);
      }
    }
    // ---- O += P V_j
    fence_regs<D / 2>(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) wgmma_rs_tb<D, T>(o, pa[kk], desc_mnmajor(aV + kk * 2048), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[stage]);      // this warp is done with K_j / V_j
    if (++stage == ST) { stage = 0; phase ^= 1; }
  }
  // ---- epilogue: row sum across the quad, O / l -> T
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_part[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? 1.f / l : 0.f;
    if constexpr (PAGED) {
      if (qrow[hh] < n) {
        T* dst = reinterpret_cast<T*>(p.o) + (long long)(qoff + qrow[hh]) * p.o_rs + (long long)h * D + 2 * t;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 8 * jj) = ElemT<T>::pack2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
      }
    } else if (qrow[hh] < p.Sq) {
      T* dst = reinterpret_cast<T*>(p.o) + (long long)b * p.o_bs + (long long)qrow[hh] * p.o_rs + (long long)h * D + 2 * t;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = ElemT<T>::pack2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

template <int D, int NWG, typename T>
__global__ void __launch_bounds__(128 * (NWG + 1), 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                  const AttnTcParams p) {
  attn_wgmma_body<D, NWG, T>(tmQ, tmK, tmV, p);
}

template <int D, int NWG, typename T>
__global__ void __launch_bounds__(128 * (NWG + 1), 1)
attn_chunk_paged_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV, const ChunkAttnParams p) {
  attn_wgmma_body<D, NWG, T>(tmQ, tmKV, tmKV, p);
}

// ---------------------------------------------------------------- host
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  });
  return fn;
}

// 3-D view [B][S][cols] of a strided 2-byte activation; box = {64 cols, box_rows rows, 1}; rows >= S are zero-filled
int make_map3(CUtensorMap* out, const void* base, long long cols, long long S, long long B, long long row_stride, long long batch_stride,
              int box_rows, CUtensorMapDataType dtype) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { vsb_set_error("cuTensorMapEncodeTiled entry point not available"); return VSB_ERR_CUDA; }
  cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)S, (cuuint64_t)B};
  cuuint64_t gstr[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)batch_stride * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, dtype, 3, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    vsb_set_error("cuTensorMapEncodeTiled(3d) failed (%d): base=%p cols=%lld S=%lld B=%lld rs=%lld bs=%lld", (int)r, base, cols, S, B,
                  row_stride, batch_stride);
    return VSB_ERR_CUDA;
  }
  return VSB_OK;
}

template <int D, int NWG, typename T>
int launch(const void* q, const CUtensorMap& tk, const CUtensorMap& tv, long long q_rs, long long q_bs, const AttnTcParams& p, int B,
           cudaStream_t st) {
  using L = ASmem<D, NWG>;
  CUtensorMap tq;
  int r = make_map3(&tq, q, (long long)p.H * D, p.Sq, B, q_rs, q_bs, 64 * NWG, ElemT<T>::tma);
  if (r) return r;
  static bool set = false;
  if (!set) { VSB_CUDA(cudaFuncSetAttribute(attn_wgmma_kernel<D, NWG, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL)); set = true; }
  dim3 grid((p.Sq + 64 * NWG - 1) / (64 * NWG), p.H, B);
  attn_wgmma_kernel<D, NWG, T><<<grid, 128 * (NWG + 1), L::TOTAL, st>>>(tq, tk, tv, p);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

}  // namespace

static int g_tc_variant = 0;    // 0 auto (two query warpgroups per CTA sharing each K/V block), 1 = one warpgroup per CTA only
void vsb_attn_tc_set_variant(int v) { g_tc_variant = v; }

// same contract as vsb_flash_attn_bf16 / vsb_flash_attn_f16 (called by them for the shapes this kernel covers)
template <typename T>
int vsb_flash_attn_tc(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs, long long k_rs,
                      long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, int D, int causal,
                      float scale, cudaStream_t stream) {
  // tensor maps cover [B][S][H*D] starting at the head-0 column of q / k / v
  CUtensorMap tk, tv;
  int r = make_map3(&tk, k, (long long)H * D, Sk, B, k_rs, k_bs, BKV, ElemT<T>::tma);
  if (r) return r;
  r = make_map3(&tv, v, (long long)H * D, Sk, B, v_rs, v_bs, BKV, ElemT<T>::tma);
  if (r) return r;
  AttnTcParams p;
  p.o = o; p.o_bs = o_bs; p.o_rs = o_rs;
  p.H = H; p.Sq = Sq; p.Sk = Sk; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  const bool two = g_tc_variant != 1 && Sq > 64;
  if (D == 64) return two ? launch<64, 2, T>(q, tk, tv, q_rs, q_bs, p, B, stream) : launch<64, 1, T>(q, tk, tv, q_rs, q_bs, p, B, stream);
  return two ? launch<128, 2, T>(q, tk, tv, q_rs, q_bs, p, B, stream) : launch<128, 1, T>(q, tk, tv, q_rs, q_bs, p, B, stream);
}
template int vsb_flash_attn_tc<bf16>(const void*, const void*, const void*, void*, long long, long long, long long, long long, long long,
                                     long long, long long, long long, int, int, int, int, int, int, float, cudaStream_t);
template int vsb_flash_attn_tc<half>(const void*, const void*, const void*, void*, long long, long long, long long, long long, long long,
                                     long long, long long, long long, int, int, int, int, int, int, float, cudaStream_t);

// ---------------------------------------------------------------- paged chunk prefill
namespace {

template <int D, int NWG, typename T>
int launch_chunk(const void* q, long long ldq, int R, const CUtensorMap& tkv, const ChunkAttnParams& p, cudaStream_t st) {
  using L = ASmem<D, NWG>;
  CUtensorMap tq;
  int r = make_map3(&tq, q, (long long)p.H * D, R, 1, ldq, (long long)R * ldq, 64 * NWG, ElemT<T>::tma);
  if (r) return r;
  static bool set = false;
  if (!set) { VSB_CUDA(cudaFuncSetAttribute(attn_chunk_paged_kernel<D, NWG, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL)); set = true; }
  // sum over segments of ceil(n / BQ) <= ceil(R / BQ) + S tiles; the CTAs past the last tile exit at once
  dim3 grid((R + 64 * NWG - 1) / (64 * NWG) + p.S, p.H);
  attn_chunk_paged_kernel<D, NWG, T><<<grid, 128 * (NWG + 1), L::TOTAL, st>>>(tq, tkv, p);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

}  // namespace

// tensor map over a pool of `rows` k|v rows of `cols` 2-byte elements (boxes of 64 rows): one map serves every layer of a pool
int vsb_pool_map(CUtensorMap* map, const void* pool, long long rows, long long cols, int f16) {
  VSB_CHECK_ARG(pool && rows > 0 && rows < (1LL << 31) && cols % 64 == 0, "vsb_attn_chunk_paged: pool of %lld rows x %lld columns", rows, cols);
  VSB_CHECK_ARG((reinterpret_cast<uintptr_t>(pool) & 15) == 0, "vsb_attn_chunk_paged: pool must be 16-byte aligned");
  return make_map3(map, pool, cols, rows, 1, cols, rows * cols, 64, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
}

// the refusals of vsb_attn_chunk_paged, before any launch
int vsb_attn_chunk_check(const void* q, long long ldq, void* o, long long ldo, int page_rows, const void* page_table, int pt_ld,
                         const void* seg, int S, int R, int H, int D) {
  VSB_CHECK_ARG(q && o && page_table && seg, "vsb_attn_chunk_paged: null pointer");
  VSB_CHECK_ARG(D == 64 || D == 128, "vsb_attn_chunk_paged: head_dim %d unsupported (64/128)", D);
  VSB_CHECK_ARG(S > 0 && R > 0 && H > 0 && pt_ld > 0, "vsb_attn_chunk_paged: bad shape (S=%d, R=%d, H=%d, pt_ld=%d)", S, R, H, pt_ld);
  VSB_CHECK_ARG(page_rows >= 64 && page_rows % 64 == 0, "vsb_attn_chunk_paged: page_rows %d is not a multiple of 64", page_rows);
  VSB_CHECK_ARG((long long)pt_ld * page_rows < (1LL << 30), "vsb_attn_chunk_paged: %d pages of %d rows per page-table row", pt_ld, page_rows);
  VSB_CHECK_ARG(ldq >= (long long)H * D && ldo >= (long long)H * D && ldq % 8 == 0 && ldo % 2 == 0 &&
                    (reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(o) & 3) == 0,
                "vsb_attn_chunk_paged: q must be 16-byte aligned with a row stride of 8k elements, o 4-byte aligned");
  return VSB_OK;
}

// causal attention of R chunk rows in S segments over paged keys (see vsb_attn_chunk_paged); the pool's map `tkv` from
// vsb_pool_map, its rows from row0 on the layer's
template <typename T>
int vsb_attn_chunk_paged_tc(const void* q, long long ldq, const CUtensorMap& tkv, long long row0, int d, void* o, long long ldo, int page_rows,
                            const void* page_table, int pt_ld, const void* seg, int S, int R, int H, int D, float scale, cudaStream_t stream) {
  ChunkAttnParams p;
  p.o = o; p.o_rs = ldo;
  p.seg = reinterpret_cast<const int*>(seg);
  p.page_table = reinterpret_cast<const int*>(page_table);
  p.S = S; p.H = H; p.pt_ld = pt_ld; p.page_rows = page_rows; p.row0 = (int)row0; p.d = d;
  p.scale_log2 = scale * 1.4426950408889634f;
  const bool two = R > 64;
  if (D == 64) return two ? launch_chunk<64, 2, T>(q, ldq, R, tkv, p, stream) : launch_chunk<64, 1, T>(q, ldq, R, tkv, p, stream);
  return two ? launch_chunk<128, 2, T>(q, ldq, R, tkv, p, stream) : launch_chunk<128, 1, T>(q, ldq, R, tkv, p, stream);
}
template int vsb_attn_chunk_paged_tc<bf16>(const void*, long long, const CUtensorMap&, long long, int, void*, long long, int, const void*, int,
                                           const void*, int, int, int, int, float, cudaStream_t);
template int vsb_attn_chunk_paged_tc<half>(const void*, long long, const CUtensorMap&, long long, int, void*, long long, int, const void*, int,
                                           const void*, int, int, int, int, float, cudaStream_t);

extern "C" int vsb_attn_chunk_paged(const void* q, long long ldq, const void* pool, long long pool_rows, long long row0, void* o, long long ldo,
                                    int page_rows, const void* page_table_i32, int pt_ld, const void* seg_i32, int S, int R, int H, int D,
                                    float scale, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_attn_chunk_paged: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  int r = vsb_attn_chunk_check(q, ldq, o, ldo, page_rows, page_table_i32, pt_ld, seg_i32, S, R, H, D);
  if (r) return r;
  VSB_CHECK_ARG(row0 >= 0 && row0 % page_rows == 0 && row0 < pool_rows, "vsb_attn_chunk_paged: row0 %lld outside the pool's %lld rows", row0,
                pool_rows);
  CUtensorMap tkv;
  r = vsb_pool_map(&tkv, pool, pool_rows, 2LL * H * D, dtype == VSB_DTYPE_F16);
  if (r) return r;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return dtype == VSB_DTYPE_F16 ? vsb_attn_chunk_paged_tc<half>(q, ldq, tkv, row0, H * D, o, ldo, page_rows, page_table_i32, pt_ld, seg_i32, S, R, H,
                                                                D, scale, st)
                                : vsb_attn_chunk_paged_tc<bf16>(q, ldq, tkv, row0, H * D, o, ldo, page_rows, page_table_i32, pt_ld, seg_i32, S, R, H,
                                                                D, scale, st);
}
