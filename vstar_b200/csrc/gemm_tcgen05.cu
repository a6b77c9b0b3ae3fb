// vsb_gemm_bf16 / vsb_gemm_f16: C[M,N] = epilogue(A[M,K] . W[N,K]^T + bias) (+ residual)
//
// Hand-written sm_90a GEMM: TMA (cp.async.bulk.tensor, 128B swizzle) -> shared
// memory ring (mbarrier full / empty pairs) -> wgmma.mma_async (bf16 or f16 ->
// fp32 in registers) -> epilogue from the accumulator registers
// (bias / activation / SwiGLU / residual / row remap / folded RMSNorm / RoPE) ->
// per-warp shared-memory slots -> global by bulk copies, one per row (T output
// with 16-byte aligned rows; fp32 output and BN = 32 store directly).  Persistent: one CTA per SM loops over 128 x BN output tiles; the
// producer keeps loading the next tile's k-blocks while the consumers run the
// epilogue of the current one.
//
// This one kernel carries every nn.Linear on the hot path (reference op sites
// H1-H3, H5, H6, H8-H10, H12-H15 of SURVEY.md §2b): CLIP/OWL patch-embed
// (as im2col GEMM), all ViT and Llama projections, the LLaVA mm_projector,
// lm_head, the [LOC]-row MLPs, OWL class/box heads and the SAM decoder linears
// and 3x3 convs (im2col).
//
// Warp groups (384 threads): warpgroup 0 = producer, minimal register budget: thread 0 issues the TMA loads, warps 1-3
// compute the folded-RMSNorm row scales of the tile the consumers finish next; warpgroups 1 and 2 = consumers: consumer c
// issues m64nBNk16 wgmma on rows [64c, 64c + 64) of the tile and stores them, reading each 32-column chunk's bias / residual
// before the previous chunk's stores.
#include "common.cuh"
#include "vstar_b200.h"
#include "wgmma.cuh"

#include <mutex>
#include <unordered_map>

namespace {

constexpr int BM = 128;
constexpr int BK = 64;   // 64 bf16 = 128 B = one swizzle-128B row
constexpr int WG_K = 16;

template <typename T>      // operand type: bf16 or half
struct GemmParams {
  void* C;
  const T* bias;
  const void* residual;
  long long ldc, ldr;
  int M, N, K;
  int epilogue;        // VSB_EPI_*
  int out_fp32;        // C (and residual) element type: 0 T (bf16 / f16), 1 fp32
  int vec2;            // C (and residual) rows allow 2-element vector access at even columns
  int staged;          // T output written through shared memory with bulk copies (16-byte aligned rows, see gemm_dispatch)
  int rows_per_group;  // output row remap: r = (m / rpg) * group_stride + group_offset + m % rpg
  long long group_stride, group_offset;
  int tiles_m, tiles_n;
  int group_m;         // tile rasterisation band height (in m-blocks)
  // L2 eviction priorities of the A / W tile loads (0 = none) and streaming (.cs) output stores, see vsb_gemm_set_l2_hints
  unsigned long long hint_a, hint_b;
  int stream_out;
  // RMSNorm folded into the GEMM (LlamaRMSNorm with its weight pre-multiplied into W, see vsb_gemm_rowscale_bf16):
  //   rowsq_in  [sq_in_chunks][sq_ld] fp32: partial sums of squares of the A rows -> output row m is scaled by
  //             rsqrt(sum_c rowsq_in[c][m] * sq_inv_cols + sq_eps) before bias / activation
  //   rowsq_out [N/32][sq_ld] fp32: sum of squares of the 32 bf16 OUTPUT values (after residual) of chunk n0/32 of row m
  const float* rowsq_in;
  float* rowsq_out;
  long long sq_ld;
  int sq_in_chunks;
  float sq_inv_cols, sq_eps;
  // rotate-half RoPE applied by the epilogue to the output columns [0, rope_cols) (the q | k thirds of a fused QKV projection,
  // heads of 128 columns): same T arithmetic as rope_kernel (elementwise.cu) on the same T GEMM results => identical bits
  const T* rope_cos;          // [max_pos][64] T
  const T* rope_sin;
  const int* rope_pos;        // optional position of every A row; else rope_pos0 + m % rope_T
  int rope_T, rope_pos0, rope_cols;
};

// ---------------------------------------------------------------- PTX wrappers
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
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(addr),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// cute::TMA::CacheHintSm90 encodings of createpolicy.fractional.L2::evict_{first,last}.b64 (fraction 1.0)
constexpr unsigned long long L2_EVICT_FIRST = 0x12F0000000000000ull;
constexpr unsigned long long L2_EVICT_LAST = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar, unsigned long long hint = 0) {
  if (hint)
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
  else
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

// bulk (non-tensor) shared -> global copies of the staged epilogue: `bytes` and both addresses multiples of 16
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_store(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t saddr, uint16_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(saddr), "h"(v) : "memory"); }
__device__ __forceinline__ void sts_u32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk group of this thread but the newest N has finished reading its shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every bulk group of this thread has completed (its global writes included)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// K-major, 128B-swizzled shared-memory operand descriptor (cute::GMMA::GmmaDescriptor):
//   [0,14) start>>4 | [16,30) LBO>>4 (=1, unused for swizzled K-major) | [32,46) SBO>>4 (8 rows * 128 B = 1024)
//   [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

constexpr int RSTD_THREADS = 96;    // warps 1-3 of the producer warpgroup: folded-RMSNorm row scales (tile_rstd)
constexpr int RSTD_PIECE = 16;      // rowsq_in chunks staged per round trip

// Staged epilogue output: each consumer warp owns two slots of its 16 rows x one 32-column chunk (T), rows OUT_PITCH bytes
// apart.  80 B = 20 banks: the 4-byte fragment writes of one instruction (8 rows x 4 lanes, banks 20r + 4jj + t mod 32) are
// conflict-free, and every row starts 16-byte aligned for its bulk copy.
constexpr int OUT_PITCH = 80;
constexpr int OUT_SLOT = 16 * OUT_PITCH;
constexpr int SMEM_OPTIN_MAX = 232448;   // H100 opt-in dynamic shared memory per block

template <int BN>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : (BN == 64 ? 8 : 10));
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int RSTD_OFFSET = BAR_OFFSET + 256;   // float [2][BM]: folded-RMSNorm row scales, two tiles in flight
  static constexpr int PART_OFFSET = RSTD_OFFSET + 2 * BM * 4;   // float [RSTD_PIECE][BM]: staged partial sums (tile_rstd)
  static constexpr int OUT_OFFSET = PART_OFFSET + RSTD_PIECE * BM * 4;   // [8 consumer warps][2][OUT_SLOT]: staged output
  // BN = 32 (batched decode, HBM-bound on W) has no room for the staging slots beside its 10 stages: it stores directly
  static constexpr bool STAGED = BN != 32;
  static constexpr int TOTAL = OUT_OFFSET + (STAGED ? 8 * 2 * OUT_SLOT : 0) + 1024;  // + alignment slack
  static_assert((2 * STAGES + 4) * 8 <= 256, "barriers overflow their 256-byte slot");
  static_assert(TOTAL <= SMEM_OPTIN_MAX, "shared memory over the per-block limit");
};

__device__ __forceinline__ float apply_act(float x, int epi) {
  switch (epi) {
    case VSB_EPI_QUICK_GELU: return quick_gelu_f(x);
    case VSB_EPI_GELU: return gelu_erf_f(x);
    case VSB_EPI_RELU: return fmaxf(x, 0.f);
    default: return x;
  }
}

// tile rasterisation: groups of GROUP_M m-blocks x all n-blocks, m fastest inside a group, so that the CTAs running
// concurrently share both A and W tiles in L2 (instead of one W tile and 132 distinct A tiles)
__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& m_blk, int& n_blk) {
  const int per_group = group_m * tiles_n;
  const int g = t / per_group;
  const int first_m = g * group_m;
  const int gsize = min(group_m, tiles_m - first_m);
  const int r = t - g * per_group;
  m_blk = first_m + r % gsize;
  n_blk = r / gsize;
}

template <typename T>
__device__ __forceinline__ long long remap_row(const GemmParams<T>& p, int m) {
  return (long long)(m / p.rows_per_group) * p.group_stride + p.group_offset + (m % p.rows_per_group);
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// 1 / rms of the BM rows of m-block m_blk from the partial sums a producer GEMM (or vsb_rowsq_bf16) left behind:
// out[r] = rsqrt(sum_c rowsq_in[c][m] * sq_inv_cols + sq_eps), summed in fp32 from 0 over c = 0 .. sq_in_chunks - 1 in order;
// 1 for rows >= M.  Run by the producer warpgroup's warps 1-3, thread r0 taking rows r0 and r0 + RSTD_THREADS.  The partials
// are staged through `part` by cp.async, RSTD_PIECE chunks per round trip: under the producer's 40-register budget plain loads
// keep only 2-3 in flight, and the sum of 128 chunks then outlasts a tile's main loop.  Each thread reads back only what it copied.
template <typename T>
__device__ __forceinline__ void tile_rstd(const GemmParams<T>& p, int m_blk, int r0, float* part, float* out) {
  const int r[2] = {r0, r0 + RSTD_THREADS};
  const bool ok[2] = {m_blk * BM + r[0] < p.M, r[1] < BM && m_blk * BM + r[1] < p.M};
  float s[2] = {0.f, 0.f};
  for (int c0 = 0; c0 < p.sq_in_chunks; c0 += RSTD_PIECE) {
    const int nc = min(RSTD_PIECE, p.sq_in_chunks - c0);
    for (int i = 0; i < nc; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (ok[h]) cp_async4(part + i * BM + r[h], p.rowsq_in + (long long)(c0 + i) * p.sq_ld + m_blk * BM + r[h]);
    cp_async_wait_all();
    for (int i = 0; i < nc; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (ok[h]) s[h] += part[i * BM + r[h]];
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (r[h] < BM) out[r[h]] = ok[h] ? rsqrtf(s[h] * p.sq_inv_cols + p.sq_eps) : 1.f;
}

// ---------------------------------------------------------------- epilogue of one accumulator pair
// Bias and residual of one accumulator pair (row orow, columns n, n+1), as fp32.  The epilogue reads them a 32-column chunk
// ahead of its stores: C, bias and residual may alias (the o-proj and down-proj GEMMs add in place, residual == C), so a load
// written after a store is issued after it, and a chain of load -> add -> store per pair would expose one memory round trip
// per pair.  Each element is still read before it is written, by the same thread.
struct PairIn {
  float b0, b1, r0, r1;
};

template <typename T>
__device__ __forceinline__ PairIn load_pair(const GemmParams<T>& p, long long orow, int n) {
  using E = ElemT<T>;
  const bool has1 = n + 1 < p.N;
  PairIn in{0.f, 0.f, 0.f, 0.f};
  if (p.bias != nullptr) {
    in.b0 = E::to_f(p.bias[n]);
    if (has1) in.b1 = E::to_f(p.bias[n + 1]);
  }
  if (p.residual == nullptr) return in;
  if (p.out_fp32) {
    const float* r = reinterpret_cast<const float*>(p.residual) + orow * p.ldr + n;
    if (has1 && p.vec2) {
      const float2 rv = *reinterpret_cast<const float2*>(r);
      in.r0 = rv.x;
      in.r1 = rv.y;
    } else {
      in.r0 = r[0];
      if (has1) in.r1 = r[1];
    }
  } else {
    const T* r = reinterpret_cast<const T*>(p.residual) + orow * p.ldr + n;
    if (has1 && p.vec2) {
      const float2 rv = E::unpack2(*reinterpret_cast<const uint32_t*>(r));
      in.r0 = rv.x;
      in.r1 = rv.y;
    } else {
      in.r0 = E::to_f(r[0]);
      if (has1) in.r1 = E::to_f(r[1]);
    }
  }
  return in;
}

// row orow (already remapped), columns n, n+1 (n even, n < N): bias -> activation / SwiGLU -> (+residual) -> T / fp32 store,
// with bias and residual from load_pair.  Returns the sum of squares of the T values stored (the folded-RMSNorm row statistics).
// STAGED: the T values go to the shared-memory staging slot at shared address s (output column n, or n/2 for SwiGLU) instead
// of C; there N % 8 == 0, so n + 1 < N.
template <bool STAGED, typename T>
__device__ __forceinline__ float epilogue_pair(const GemmParams<T>& p, long long orow, int n, float x0, float x1, bool swiglu,
                                               const PairIn& in, uint32_t s) {
  using E = ElemT<T>;
  const bool has1 = n + 1 < p.N;
  if (p.bias != nullptr) {
    x0 += in.b0;
    if (has1) x1 += in.b1;
  }
  if (swiglu) {
    // interleaved weight rows: even column = gate_j, odd column = up_j -> out column n/2 (N is even)
    const T v = E::from_f(silu_f(x0) * x1);
    if constexpr (STAGED) sts_u16(s, *reinterpret_cast<const uint16_t*>(&v));
    else reinterpret_cast<T*>(p.C)[orow * p.ldc + (n >> 1)] = v;
    return 0.f;
  }
  x0 = apply_act(x0, p.epilogue);
  x1 = apply_act(x1, p.epilogue);
  if (p.residual != nullptr) {
    x0 += in.r0;
    if (has1) x1 += in.r1;
  }
  if constexpr (STAGED) {
    sts_u32(s, E::pack2(x0, x1));
    const float s0 = E::round(x0), s1 = E::round(x1);
    return fmaf(s1, s1, s0 * s0);
  }
  if (p.out_fp32) {
    float* c = reinterpret_cast<float*>(p.C) + orow * p.ldc + n;
    if (has1 && p.vec2) {
      *reinterpret_cast<float2*>(c) = make_float2(x0, x1);
    } else {
      c[0] = x0;
      if (has1) c[1] = x1;
    }
    return 0.f;
  }
  T* c = reinterpret_cast<T*>(p.C) + orow * p.ldc + n;
  if (has1 && p.vec2) {
    const uint32_t w = E::pack2(x0, x1);
    if (p.stream_out) __stcs(reinterpret_cast<unsigned int*>(c), w); else *reinterpret_cast<uint32_t*>(c) = w;
  } else {
    c[0] = E::from_f(x0);
    if (has1) c[1] = E::from_f(x1);
  }
  const float s0 = E::round(x0), s1 = has1 ? E::round(x1) : 0.f;
  return fmaf(s1, s1, s0 * s0);
}

// RoPE on a 256-wide q/k tile (two heads of 128): accumulator column i of a head (i < 64) pairs with column i + 64, i.e.
// fragment block j with j + 8.  x = T(acc * rs) is what the un-fused path stores and rope_kernel reads back; the rotated
// values are exactly representable in T (the store path's rounding is then the identity).
template <typename T>
__device__ __forceinline__ void rope_tile(const GemmParams<T>& p, float* acc, const int* m, const float* rs, int t) {
  using E = ElemT<T>;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int pos = (m[h] < p.M) ? (p.rope_pos ? p.rope_pos[m[h]] : p.rope_pos0 + (m[h] % p.rope_T)) : 0;
    const T* cr = p.rope_cos + (long long)pos * 64;
    const T* sr = p.rope_sin + (long long)pos * 64;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int i = 8 * jj + 2 * t;
      const float2 cs = E::unpack2(__ldg(reinterpret_cast<const unsigned int*>(cr + i)));
      const float2 sn = E::unpack2(__ldg(reinterpret_cast<const unsigned int*>(sr + i)));
#pragma unroll
      for (int head = 0; head < 2; ++head) {
        const int ja = 16 * head + jj, jb = ja + 8;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float c = e ? cs.y : cs.x, s = e ? sn.y : sn.x;
          float& a = acc[4 * ja + 2 * h + e];
          float& b = acc[4 * jb + 2 * h + e];
          const float x1 = E::round(a * rs[h]), x2 = E::round(b * rs[h]);
          a = E::round(E::round(x1 * c) + E::round(-x2 * s));
          b = E::round(E::round(x2 * c) + E::round(x1 * s));
        }
      }
    }
  }
}

// load_pair for the 8 accumulator pairs of one thread in the 32-column chunk starting at n0
template <typename T>
__device__ __forceinline__ void load_chunk(const GemmParams<T>& p, const bool* ok, const long long* orow, int n0, int t, PairIn (&in)[4][2]) {
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int n = n0 + 8 * jj + 2 * t;
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (ok[h] && n < p.N) in[jj][h] = load_pair<T>(p, orow[h], n);
  }
}

// Epilogue of one consumer thread: rows m[0], m[1] of the tile, fragment columns 8j + 2t (see wgmma.cuh); rs = their
// folded-RMSNorm scales (1 without a folded norm).
// STAGED: each 32-column chunk of the warp's 16 rows is written into one of the warp's two shared-memory slots (`stage`, slot
// `oslot & 1`, oslot counting the warp's slot fills across tiles) and leaves as one bulk copy per row, issued by lanes 0-15.
// SwiGLU halves the columns, so a slot takes the 16 output columns of two consecutive chunks and is copied after the second
// (64-byte rows, half as many copies).  The warp waits only until the copies of the fill before last have read their slot,
// never for a global write.  SW: the staged SwiGLU epilogue (a template parameter so the other epilogues keep a branch-free
// chunk loop).  In-place residual
// (C == residual) stays safe: every element's residual load completes before its value is written to the slot (the value depends
// on it), so before the bulk copy that writes the same bytes is issued, and chunk c + 1's loads touch no column of chunk c.  Tiles
// (and remapped rows) are disjoint, so no other thread reads what a copy writes.
template <int BN, bool ROPE, bool STAGED, bool SW, typename T>
__device__ __forceinline__ void epilogue_tile(const GemmParams<T>& p, float* acc, int m0, int n_blk, int t, float rs0, float rs1,
                                              uint8_t* stage, int& oslot) {
  static_assert(BN % 32 == 0, "the epilogue works in whole 32-column chunks");
  const int lane = threadIdx.x & 31;
  const int m[2] = {m0, m0 + 8};
  float rs[2] = {rs0, rs1};
  const bool ok[2] = {m[0] < p.M, m[1] < p.M};
  const long long orow[2] = {ok[0] ? remap_row(p, m[0]) : 0, ok[1] ? remap_row(p, m[1]) : 0};
  const bool swiglu = STAGED ? SW : (p.epilogue == VSB_EPI_SWIGLU);
  const int n_tile0 = n_blk * BN;
  if constexpr (ROPE) {
    if (n_tile0 < p.rope_cols) {
      rope_tile<T>(p, acc, m, rs, t);
      rs[0] = rs[1] = 1.f;
    }
  }
  // fused QKV + RoPE has neither bias nor residual (gemm_qkv_rope): no input registers beside its 128 accumulators
  const bool has_in = !ROPE && (p.bias != nullptr || p.residual != nullptr);
  PairIn in[2][4][2];                              // chunk c uses in[c & 1] while chunk c + 1 loads into the other half
  if (has_in) load_chunk<T>(p, ok, orow, n_tile0, t, in[0]);
#pragma unroll
  for (int c = 0; c < BN / 32; ++c) {              // 32-column chunks (the granularity of the row statistics)
    const int n0 = n_tile0 + 32 * c;
    if (n0 >= p.N) break;                          // warp-uniform
    if (has_in && c + 1 < BN / 32 && n0 + 32 < p.N) load_chunk<T>(p, ok, orow, n0 + 32, t, in[(c + 1) & 1]);
    uint8_t* slot = stage + (oslot & 1) * OUT_SLOT;    // the warp's staging slot for this chunk
    const int half = SW ? (c & 1) : 0;             // SwiGLU: second chunk of the slot's two
    if (STAGED && half == 0) {
      bulk_wait_read<1>();                         // the copies that last read this slot (fill before last) are done with it
      __syncwarp();
    }
    float sq[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;
      const int n = n0 + 8 * jj + 2 * t;
      const int sc = swiglu ? 16 * half + 4 * jj + t : 8 * jj + 2 * t;   // column in the slot
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (ok[h] && n < p.N)
          sq[h] += epilogue_pair<STAGED, T>(p, orow[h], n, acc[4 * j + 2 * h] * rs[h], acc[4 * j + 2 * h + 1] * rs[h], swiglu,
                                            in[c & 1][jj][h], smem_u32(slot) + (8 * h + (lane >> 2)) * OUT_PITCH + sc * (int)sizeof(T));
    }
    if (STAGED && (!SW || half == 1 || n0 + 32 >= p.N)) {
      fence_proxy_async_smem();                    // this thread's slot writes -> visible to the bulk copies
      __syncwarp();
      const int mr = m0 - (lane >> 2) + lane;      // lane < 16: tile row of slot row `lane`
      if (lane < 16 && mr < p.M) {
        const int nb = n0 - 32 * half;             // first input column of the slot
        // bytes: 2 per output column; the output width is a multiple of 8 on this path
        const int bytes = swiglu ? min(64, p.N - nb) : 2 * min(32, p.N - nb);
        T* dst = reinterpret_cast<T*>(p.C) + remap_row(p, mr) * p.ldc + (swiglu ? nb >> 1 : nb);
        bulk_store(dst, slot + lane * OUT_PITCH, bytes);
      }
      bulk_commit();
      ++oslot;
    }
    if (p.rowsq_out != nullptr) {                  // N % 32 == 0: every chunk is complete
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 1);
        sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 2);
        if (t == 0 && ok[h]) p.rowsq_out[(long long)(n0 >> 5) * p.sq_ld + orow[h]] = sq[h];
      }
    }
  }
}

template <int N>
__device__ __forceinline__ void fence_acc(float* acc) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

constexpr int GEMM_THREADS = 384;   // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma consumers + epilogue

template <int BN, bool ROPE, typename T>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams<T> p) {
  using L = SmemLayout<BN>;
  constexpr int STAGES = L::STAGES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* rstd_full = empty_bar + STAGES;     // [2]: the row scales of slot s are written
  uint64_t* rstd_empty = rstd_full + 2;         // [2]: every consumer thread has read them
  float* rstd_s = reinterpret_cast<float*>(smem + L::RSTD_OFFSET);   // [2][BM]

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;
  const int num_tiles = p.tiles_m * p.tiles_n;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&rstd_full[s], RSTD_THREADS);
      mbar_init(&rstd_empty[s], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(tile, p.tiles_m, p.tiles_n, p.group_m, m_blk, n_blk);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          tma_load_2d(sa, &tmA, kb * BK, m_blk * BM, &full_bar[stage], p.hint_a);
          tma_load_2d(sb, &tmB, kb * BK, n_blk * BN, &full_bar[stage], p.hint_b);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (threadIdx.x >= 32 && p.rowsq_in != nullptr) {
      // warps 1-3: the folded-RMSNorm scale of each row of the tiles this CTA runs, one tile ahead of the consumers' epilogue
      // (each row sum reads sq_in_chunks scattered floats; in the epilogue that latency would stall the tensor cores)
      float* part = reinterpret_cast<float*>(smem + L::PART_OFFSET);
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        int m_blk, n_blk;
        tile_coords(tile, p.tiles_m, p.tiles_n, p.group_m, m_blk, n_blk);
        const int slot = it & 1;
        mbar_wait(&rstd_empty[slot], ((it >> 1) & 1) ^ 1);
        tile_rstd(p, m_blk, threadIdx.x - 32, part, rstd_s + slot * BM);
        mbar_arrive(&rstd_full[slot]);
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;                        // rows [64 cw, 64 cw + 64) of the tile
  const int wq = (threadIdx.x >> 5) & 3;        // warp inside the warpgroup: 16 rows each
  float acc[BN / 2];
  uint8_t* ostage = smem + L::OUT_OFFSET + (threadIdx.x / 32 - 4) * (2 * OUT_SLOT);   // this warp's two output slots
  int oslot = 0;
  int stage = 0;
  uint32_t phase = 0;
  int it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    int m_blk, n_blk;
    tile_coords(tile, p.tiles_m, p.tiles_n, p.group_m, m_blk, n_blk);
    int prev = -1;
    fence_acc<BN / 2>(acc);
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES) + cw * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * L::STAGE_BYTES) + L::A_BYTES;
      const uint64_t da = make_smem_desc(sa);
      const uint64_t db = make_smem_desc(sb);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WG_K; ++k)
        // advance 16 bf16 = 32 B along K inside the 128B swizzle row: +2 in the (addr>>4) field
        wgmma_ss<BN, T>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1 : 0);
      wgmma_commit();
      wgmma_wait<1>();                            // the k-block before this one has been consumed: free its stage
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc<BN / 2>(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
    const int r = cw * 64 + wq * 16 + (lane >> 2);   // tile row of the thread's first accumulator row
    float rs0 = 1.f, rs1 = 1.f;
    if (p.rowsq_in != nullptr) {
      const int slot = it & 1;
      mbar_wait(&rstd_full[slot], (it >> 1) & 1);
      rs0 = rstd_s[slot * BM + r];
      rs1 = rstd_s[slot * BM + r + 8];
      mbar_arrive(&rstd_empty[slot]);
    }
    if (L::STAGED && p.staged && !ROPE && p.epilogue == VSB_EPI_SWIGLU)
      epilogue_tile<BN, ROPE, L::STAGED, !ROPE, T>(p, acc, m_blk * BM + r, n_blk, lane & 3, rs0, rs1, ostage, oslot);
    else if (L::STAGED && p.staged)
      epilogue_tile<BN, ROPE, L::STAGED, false, T>(p, acc, m_blk * BM + r, n_blk, lane & 3, rs0, rs1, ostage, oslot);
    else
      epilogue_tile<BN, ROPE, false, false, T>(p, acc, m_blk * BM + r, n_blk, lane & 3, rs0, rs1, ostage, oslot);
  }
  bulk_wait_all();   // the staging slots must outlive the copies that read them
}

// ---------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr;
  long long rows, cols, ld;
  int box_rows;
  CUtensorMapDataType dtype;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && dtype == o.dtype;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h ^= std::hash<long long>()(k.rows * 1315423911LL + k.cols) + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
    h ^= std::hash<long long>()((k.ld * 31 + k.box_rows) * 4 + (int)k.dtype) + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
    return h;
  }
};

std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;

// 2D row-major [rows, cols] of a 2-byte type with leading dimension ld (elements); box = {64 cols, box_rows}
int make_tensor_map(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_rows, CUtensorMapDataType dtype) {
  MapKey key{ptr, rows, cols, ld, box_rows, dtype};
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) {
      *out = it->second;
      return VSB_OK;
    }
  }
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    vsb_set_error("cuTensorMapEncodeTiled entry point not available");
    return VSB_ERR_CUDA;
  }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, dtype, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    vsb_set_error("cuTensorMapEncodeTiled failed (%d) ptr=%p rows=%lld cols=%lld ld=%lld box_rows=%d", (int)r, ptr, rows,
                  cols, ld, box_rows);
    return VSB_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    if (g_map_cache.size() > 8192) g_map_cache.clear();
    g_map_cache[key] = *out;
  }
  return VSB_OK;
}

template <int BN, bool ROPE, typename T>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams<T>& p, int max_ctas, cudaStream_t stream) {
  using L = SmemLayout<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    VSB_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, ROPE, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    attr_set = true;
  }
  p.tiles_m = (p.M + BM - 1) / BM;
  p.tiles_n = (p.N + BN - 1) / BN;
  int tiles = p.tiles_m * p.tiles_n;
  int grid = tiles < max_ctas ? tiles : max_ctas;
  gemm_wgmma_kernel<BN, ROPE, T><<<grid, GEMM_THREADS, L::TOTAL, stream>>>(tmA, tmB, p);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

int g_l2_hints = 0;      // bit mask of L2 eviction hints on large GEMMs (see gemm_dispatch); 0 = none
int g_force_bn = 0;      // 32/64/128/256 = tile width; 1 / 2 = force a skinny decode kernel; 0 = auto
int g_max_ctas = 0;
int g_group_m = 0;

}  // namespace

extern "C" int vsb_gemm_set_tuning(int force_bn, int max_ctas) {
  VSB_CHECK_ARG(force_bn == 0 || force_bn == 1 || force_bn == 2 || force_bn == 32 || force_bn == 64 || force_bn == 128 || force_bn == 256,
                "vsb_gemm_set_tuning: force_bn %d is none of 0, 1, 2, 32, 64, 128, 256", force_bn);
  VSB_CHECK_ARG(max_ctas >= 0, "vsb_gemm_set_tuning: max_ctas %d < 0", max_ctas);
  g_force_bn = force_bn;
  g_max_ctas = max_ctas;
  return VSB_OK;
}
int vsb_gemm_forced_bn() { return g_force_bn; }
extern "C" int vsb_gemm_set_l2_hints(int on) {
  g_l2_hints = on;
  return VSB_OK;
}

extern "C" int vsb_gemm_set_group_m(int group_m) {
  g_group_m = group_m;
  return VSB_OK;
}

template <typename T>
int vsb_gemm_skinny_launch(int variant, const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                           int K, const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                           long long group_stride, long long group_offset, cudaStream_t stream);

// ---------------------------------------------------------------- CUDA-event profiling of every launch (bench.py roofline leg)
#include <vector>
namespace {
struct ProfRec { cudaEvent_t a, b; double flops; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
void prof_clear() {
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
}
}  // namespace

extern "C" int vsb_gemm_profile_begin(void) {
  prof_clear();
  g_prof_on = true;
  return VSB_OK;
}
extern "C" int vsb_gemm_profile_end(double* flops, double* ms, long long* launches) {
  g_prof_on = false;
  VSB_CUDA(cudaDeviceSynchronize());
  double f = 0, t = 0;
  for (auto& r : g_prof) {
    float e = 0.f;
    VSB_CUDA(cudaEventElapsedTime(&e, r.a, r.b));
    f += r.flops;
    t += e;
  }
  if (flops) *flops = f;
  if (ms) *ms = t;
  if (launches) *launches = (long long)g_prof.size();
  prof_clear();
  return VSB_OK;
}

struct RowSq {          // folded-RMSNorm side channels of a GEMM (see vsb_gemm_rowscale_bf16) + fused RoPE (vsb_gemm_qkv_rope_bf16)
  const float* in = nullptr;
  float* out = nullptr;
  long long ld = 0;
  int in_chunks = 0;
  float inv_cols = 0.f, eps = 0.f;
  const void* rope_cos = nullptr;
  const void* rope_sin = nullptr;
  const int* rope_pos = nullptr;
  int rope_T = 1, rope_pos0 = 0, rope_cols = 0;
};

template <typename T>
static int gemm_dispatch(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                         const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                         long long group_stride, long long group_offset, const RowSq* rsq, void* stream_);

template <typename T>
static int gemm_profiled(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                         const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                         long long group_stride, long long group_offset, const RowSq* rsq, void* stream_);

extern "C" int vsb_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M,
                             int N, int K, const void* bias, const void* residual, long long ldr, int epilogue,
                             int out_fp32, int rows_per_group, long long group_stride, long long group_offset,
                             void* stream_) {
  return gemm_profiled<bf16>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group, group_stride, group_offset,
                       nullptr, stream_);
}
extern "C" int vsb_gemm_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M,
                            int N, int K, const void* bias, const void* residual, long long ldr, int epilogue,
                            int out_fp32, int rows_per_group, long long group_stride, long long group_offset,
                            void* stream_) {
  return gemm_profiled<half>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group, group_stride,
                             group_offset, nullptr, stream_);
}

// GEMM with LlamaRMSNorm folded in (the norm weight must already be multiplied into W's columns):
//   rowsq_in  != NULL: C row m = epi(rsqrt(sum_c rowsq_in[c*sq_ld + m] / K + eps) * (A[m] . W^T) + bias) (+ residual), i.e. the GEMM
//                      reads the UN-normalised residual stream and applies 1/rms in its epilogue (fp32) - no norm kernel, no
//                      normalised copy of the activations
//   rowsq_out != NULL: additionally writes, for every output row and 32-column chunk, the sum of squares of the bf16 values it
//                      stored: rowsq_out[(n/32)*sq_ld + row]; the next folded GEMM consumes them with sq_in_chunks = N/32.
// T output, N % 32 == 0 when rowsq_out is given.  Always the wgmma tile kernels (any M).
template <typename T>
static int gemm_rowscale(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                      int K, const void* bias, const void* residual, long long ldr, int epilogue, int rows_per_group,
                                      long long group_stride, long long group_offset, const void* rowsq_in, int sq_in_chunks, float eps,
                                      void* rowsq_out, long long sq_ld, void* stream_) {
  VSB_CHECK_ARG(rowsq_in || rowsq_out, "vsb_gemm_rowscale_bf16: neither rowsq_in nor rowsq_out given (use vsb_gemm_bf16)");
  VSB_CHECK_ARG(sq_ld >= M && (!rowsq_in || sq_in_chunks > 0), "vsb_gemm_rowscale_bf16: bad sq_ld / sq_in_chunks");
  VSB_CHECK_ARG(!rowsq_out || (N % 32 == 0 && ldc % 8 == 0 && epilogue != VSB_EPI_SWIGLU && (reinterpret_cast<uintptr_t>(C) & 15) == 0 &&
                               (residual == nullptr || (ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(residual) & 15) == 0))),
                "vsb_gemm_rowscale_bf16: rowsq_out needs N %% 32 == 0 and 16-byte aligned bf16 rows");
  RowSq r;
  r.in = reinterpret_cast<const float*>(rowsq_in);
  r.out = reinterpret_cast<float*>(rowsq_out);
  r.ld = sq_ld;
  r.in_chunks = sq_in_chunks;
  r.inv_cols = 1.f / (float)K;
  r.eps = eps;
  return gemm_profiled<T>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, 0, rows_per_group, group_stride, group_offset, &r,
                          stream_);
}
extern "C" int vsb_gemm_rowscale_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                      int K, const void* bias, const void* residual, long long ldr, int epilogue, int rows_per_group,
                                      long long group_stride, long long group_offset, const void* rowsq_in, int sq_in_chunks, float eps,
                                      void* rowsq_out, long long sq_ld, void* stream_) {
  return gemm_rowscale<bf16>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, rows_per_group, group_stride, group_offset,
                             rowsq_in, sq_in_chunks, eps, rowsq_out, sq_ld, stream_);
}
extern "C" int vsb_gemm_rowscale_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                     int K, const void* bias, const void* residual, long long ldr, int epilogue, int rows_per_group,
                                     long long group_stride, long long group_offset, const void* rowsq_in, int sq_in_chunks, float eps,
                                     void* rowsq_out, long long sq_ld, void* stream_) {
  return gemm_rowscale<half>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, rows_per_group, group_stride, group_offset,
                             rowsq_in, sq_in_chunks, eps, rowsq_out, sq_ld, stream_);
}

// Fused QKV projection of a Llama layer: C = [q | k | v] = (A . W^T) with optional folded RMSNorm (rowsq_in, as
// vsb_gemm_rowscale_bf16) and rotate-half RoPE applied by the epilogue to the q and k thirds (columns [0, 2N/3), head_dim 128):
// the q/k rows land in the KV cache already rotated, vsb_rope_bf16 does not run.  Bit-identical to GEMM followed by vsb_rope_bf16.
template <typename T>
static int gemm_qkv_rope(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                      int K, int rows_per_group, long long group_stride, long long group_offset, const void* rowsq_in,
                                      int sq_in_chunks, float eps, long long sq_ld, const void* cos_table, const void* sin_table,
                                      const void* positions, int rope_T, int pos0, int head_dim, void* stream_) {
  VSB_CHECK_ARG(cos_table && sin_table && head_dim == 128 && rope_T > 0, "vsb_gemm_qkv_rope_bf16: head_dim must be 128 (got %d)", head_dim);
  VSB_CHECK_ARG(N % 768 == 0 && ldc % 8 == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0, "vsb_gemm_qkv_rope_bf16: N = 3*d with d %% 256 == 0");
  VSB_CHECK_ARG(!rowsq_in || (sq_in_chunks > 0 && sq_ld >= M), "vsb_gemm_qkv_rope_bf16: bad row statistics");
  RowSq r;
  r.in = reinterpret_cast<const float*>(rowsq_in);
  r.ld = sq_ld;
  r.in_chunks = sq_in_chunks;
  r.inv_cols = 1.f / (float)K;
  r.eps = eps;
  r.rope_cos = cos_table;
  r.rope_sin = sin_table;
  r.rope_pos = reinterpret_cast<const int*>(positions);
  r.rope_T = rope_T;
  r.rope_pos0 = pos0;
  r.rope_cols = N / 3 * 2;
  return gemm_profiled<T>(A, lda, W, ldw, C, ldc, M, N, K, nullptr, nullptr, 0, VSB_EPI_NONE, 0, rows_per_group, group_stride, group_offset,
                          &r, stream_);
}
extern "C" int vsb_gemm_qkv_rope_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                      int K, int rows_per_group, long long group_stride, long long group_offset, const void* rowsq_in,
                                      int sq_in_chunks, float eps, long long sq_ld, const void* cos_table, const void* sin_table,
                                      const void* positions, int T, int pos0, int head_dim, void* stream_) {
  return gemm_qkv_rope<bf16>(A, lda, W, ldw, C, ldc, M, N, K, rows_per_group, group_stride, group_offset, rowsq_in, sq_in_chunks, eps, sq_ld,
                             cos_table, sin_table, positions, T, pos0, head_dim, stream_);
}
extern "C" int vsb_gemm_qkv_rope_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                                     int K, int rows_per_group, long long group_stride, long long group_offset, const void* rowsq_in,
                                     int sq_in_chunks, float eps, long long sq_ld, const void* cos_table, const void* sin_table,
                                     const void* positions, int T, int pos0, int head_dim, void* stream_) {
  return gemm_qkv_rope<half>(A, lda, W, ldw, C, ldc, M, N, K, rows_per_group, group_stride, group_offset, rowsq_in, sq_in_chunks, eps, sq_ld,
                             cos_table, sin_table, positions, T, pos0, head_dim, stream_);
}

template <typename T>
static int gemm_profiled(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                         const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                         long long group_stride, long long group_offset, const RowSq* rsq, void* stream_) {
  if (!g_prof_on)
    return gemm_dispatch<T>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group, group_stride,
                            group_offset, rsq, stream_);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfRec r;
  VSB_CUDA(cudaEventCreate(&r.a));
  VSB_CUDA(cudaEventCreate(&r.b));
  r.flops = 2.0 * (double)M * (double)N * (double)K;
  VSB_CUDA(cudaEventRecord(r.a, stream));
  const int rc = gemm_dispatch<T>(A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group, group_stride,
                               group_offset, rsq, stream_);
  VSB_CUDA(cudaEventRecord(r.b, stream));
  g_prof.push_back(r);
  return rc;
}

template <typename T>
static int gemm_dispatch(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M,
                             int N, int K, const void* bias, const void* residual, long long ldr, int epilogue,
                             int out_fp32, int rows_per_group, long long group_stride, long long group_offset,
                             const RowSq* rsq, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  VSB_CHECK_ARG(A && W && C, "vsb_gemm_bf16: null pointer");
  VSB_CHECK_ARG(M > 0 && N > 0 && K > 0, "vsb_gemm_bf16: bad shape M=%d N=%d K=%d", M, N, K);
  VSB_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0, "vsb_gemm_bf16: lda/ldw must be multiples of 8 (TMA 16 B stride), got %lld %lld", lda, ldw);
  VSB_CHECK_ARG(lda >= K && ldw >= K, "vsb_gemm_bf16: leading dimension smaller than K");
  VSB_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
                "vsb_gemm_bf16: A/W must be 16-byte aligned");
  VSB_CHECK_ARG(epilogue >= VSB_EPI_NONE && epilogue <= VSB_EPI_SWIGLU, "vsb_gemm_bf16: bad epilogue %d", epilogue);
  VSB_CHECK_ARG(!(epilogue == VSB_EPI_SWIGLU && (out_fp32 || residual || (N & 1))), "vsb_gemm_bf16: SwiGLU epilogue is bf16 / f16, no residual, even N");
  if (rows_per_group <= 0) {
    rows_per_group = M;
    group_stride = 0;
    group_offset = 0;
  }
  GemmParams<T> p;
  p.C = C;
  p.bias = reinterpret_cast<const T*>(bias);
  p.residual = residual;
  p.ldc = ldc;
  p.ldr = ldr;
  p.M = M; p.N = N; p.K = K;
  p.epilogue = epilogue;
  p.out_fp32 = out_fp32;
  p.rows_per_group = rows_per_group;
  p.group_stride = group_stride;
  p.group_offset = group_offset;
  p.rowsq_in = rsq ? rsq->in : nullptr;
  p.rowsq_out = rsq ? rsq->out : nullptr;
  p.sq_ld = rsq ? rsq->ld : 0;
  p.sq_in_chunks = rsq ? rsq->in_chunks : 0;
  p.sq_inv_cols = rsq ? rsq->inv_cols : 0.f;
  p.sq_eps = rsq ? rsq->eps : 0.f;
  p.rope_cos = rsq ? reinterpret_cast<const T*>(rsq->rope_cos) : nullptr;
  p.rope_sin = rsq ? reinterpret_cast<const T*>(rsq->rope_sin) : nullptr;
  p.rope_pos = rsq ? rsq->rope_pos : nullptr;
  p.rope_T = rsq ? rsq->rope_T : 1;
  p.rope_pos0 = rsq ? rsq->rope_pos0 : 0;
  p.rope_cols = rsq ? rsq->rope_cols : 0;

  // decode-sized problems are HBM-bound on W: weight-streaming kernels (gemm_skinny.cu): the FMA kernel at M = 1, the mma.sync
  // kernel up to M = 8 (up to M = 16 when N <= 8192); force_bn = 1 / 2 forces one of them (tests)
  if ((K % 8) == 0 && !(vsb_batch_invariant() && g_force_bn == 0) && rsq == nullptr) {
    int variant = 0;
    if (g_force_bn == 1 && M <= 8) variant = 1;
    else if (g_force_bn == 2 && M <= 16) variant = 2;
    else if (g_force_bn == 0 && M == 1) variant = 1;
    else if (g_force_bn == 0 && (M <= 8 || (M <= 16 && N <= 8192))) variant = 2;
    if (variant)
      return vsb_gemm_skinny_launch<T>(variant, A, lda, W, ldw, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group,
                                    group_stride, group_offset, stream);
  }
  VSB_CHECK_ARG(g_force_bn != 1 && g_force_bn != 2, "vsb_gemm_bf16: skinny kernel forced but M=%d too large or K %% 8 != 0", M);
  const int sms = g_max_ctas > 0 ? g_max_ctas : vsb_num_sms();
  // tile-width choice: minimise (waves * BN) ~ time; prefer the wider tile on ties (less A re-streaming).  256-wide tiles only
  // for SwiGLU (and the fused RoPE, below): with every other epilogue a 256-wide tile writes 256 output columns per tile row,
  // and on H100 its fixed cost per wave (~39 us against ~18 us at BN = 128) and its main-loop rate (~410 against ~715 TFLOP/s)
  // make it slower than two 128-wide tiles at the same waves * BN (e.g. OWL-B qkv, M = 18440, N = 2304, K = 768: 0.49 -> 0.34 ms)
  int bn = 64;
  if (g_force_bn) {
    bn = g_force_bn;
  } else if (N > 64) {
    const int tm = (M + BM - 1) / BM;
    long long best = -1;
    const int cands[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
      int c = cands[i];
      if (c == 256 && epilogue != VSB_EPI_SWIGLU) continue;
      if (c == 64 && N > 512) continue;
      long long tiles = (long long)tm * ((N + c - 1) / c);
      long long waves = (tiles + sms - 1) / sms;
      long long cost = waves * c;
      if (best < 0 || cost < best) { best = cost; bn = c; }
    }
  }
  // batched decode (M <= 128) on the N = 4096 projections: 64-wide tiles give only 64 CTAs, each streaming a long K; 32-wide
  // tiles put twice as many SMs on the weight stream (the problem is HBM-bound on W)
  if (g_force_bn == 0 && bn == 64 && (long long)((M + BM - 1) / BM) * ((N + 63) / 64) <= sms / 2 && N >= 64) bn = 32;
  p.group_m = g_group_m > 0 ? g_group_m : 16;      // 2048-row bands (single-CTA tiles)
  CUtensorMap tmA, tmB;
  int r = make_tensor_map(&tmA, A, M, K, lda, BM, ElemT<T>::tma);
  if (r) return r;
  p.hint_a = p.hint_b = 0;
  p.stream_out = 0;
  if (g_force_bn == 0 && M >= 512 && N >= 512 && K >= 1024) {
    // large GEMMs, optional L2 policy (vsb_gemm_set_l2_hints): bit 0: A tiles evict_last (the band of A rows is re-read by every
    // n-block of its raster group), bit 1: W tiles evict_first, bit 3: W tiles evict_last, bit 2: output stores with .cs semantics
    if (g_l2_hints & 1) p.hint_a = L2_EVICT_LAST;
    if (g_l2_hints & 2) p.hint_b = L2_EVICT_FIRST;
    if (g_l2_hints & 8) p.hint_b = L2_EVICT_LAST;
    if (g_l2_hints & 4) p.stream_out = 1;
  }
  // 2-element (4 / 8 byte) vector access to C and the residual at even columns
  const int esz = out_fp32 ? 4 : 2;
  p.vec2 = (ldc % 2 == 0) && (reinterpret_cast<uintptr_t>(C) % (2 * esz) == 0) &&
           (residual == nullptr || ((ldr % 2 == 0) && (reinterpret_cast<uintptr_t>(residual) % (2 * esz) == 0)));
  if (p.rope_cos != nullptr) bn = 256;        // the fused-RoPE epilogue pairs columns inside one 128-wide head: 256-wide tiles only
  // staged epilogue (T output through shared memory, one bulk copy per row and 32-column chunk): needs 16-byte aligned rows and
  // chunks.  fp32 output (its rows would need twice the staging), the BN = 32 tiles (no room beside their stages) and the
  // streaming-store switch (.cs stores, vsb_gemm_set_l2_hints bit 2) store straight from the registers.
  const int out_cols = epilogue == VSB_EPI_SWIGLU ? N / 2 : N;
  p.staged = !out_fp32 && bn != 32 && !p.stream_out && (ldc * esz) % 16 == 0 && reinterpret_cast<uintptr_t>(C) % 16 == 0 &&
             out_cols % 8 == 0;
  r = make_tensor_map(&tmB, W, N, K, ldw, bn, ElemT<T>::tma);
  if (r) return r;
  if (bn == 256)
    return p.rope_cos ? launch_gemm<256, true, T>(tmA, tmB, p, sms, stream) : launch_gemm<256, false, T>(tmA, tmB, p, sms, stream);
  if (bn == 128) return launch_gemm<128, false, T>(tmA, tmB, p, sms, stream);
  if (bn == 32) return launch_gemm<32, false, T>(tmA, tmB, p, sms, stream);
  return launch_gemm<64, false, T>(tmA, tmB, p, sms, stream);
}
