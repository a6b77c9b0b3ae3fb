// Beam search of the SEAL VQA LLM (free_form_inference(num_beams = k), HF `beam_search` of transformers 4.31 as restated in
// oracle/beam_oracle.py): the per-step candidate selection and the KV-cache row copies that reorder the beams.
//
// vsb_beam_candidates_f32: one CTA per request.  For each of the request's k_in rows (cache-slot rows of the logits):
//   logp_i = dtype(x_i - max - log sum_j exp(x_j - max)), x = float(dtype(logit)), the sum in fp64 over fp32 exp terms and the
//   difference in fp64, rounded once to dtype; candidate score s = float(logp_i) + beam_score in fp32.
// The 2k largest s over the request's k_in * V candidates, ties by ascending flattened index beam * V + token, are found by a
// four-pass 8-bit radix select on the 32-bit order-preserving key of s (radix_select.cuh), so equal fp32 sums of distinct
// log-probs tie exactly as they do in the oracle.  The candidates at or above the threshold are compacted into shared memory
// and bitonic-sorted by (key desc, index asc); a tie at the threshold wider than that buffer is resolved by one ordered pass.
//
// vsb_copy_cache_rows_b16 / vsb_copy_slot_rows_b16: rows of the fused-QKV cache [L][B, Tmax, 3d] from slot src to slot dst for
// every layer and every pair, in one launch; one row range [lo, hi) for all pairs, or each pair's own (a decode stream, where
// every beam request forks at its own length).  Pairs travel in the kernel's parameters; a slot that is both a source and a
// destination (or two pairs with one destination) is refused, so no CTA reads a row another CTA writes.
//
// vsb_copy_page_rows_b16: the same ranged copy into a paged KV pool, each row's page found through the page table; the source is
// the pool itself (a beam fork) or a contiguous cache (a prefilled prompt's k|v rows written into its pages at admission).
//
// vsb_swap_pages_b16: whole pages of every layer between the pool and a swap area of pinned host memory, which the kernel reads
// and writes through its mapped device address in 16-byte vectors (a preempted request of a growing paged stream).  Pairs
// travel in the kernel's parameters, VSB_SWAP_PAGES_PER_LAUNCH per launch; the whole list is checked before the first launch.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "radix_select.cuh"
#include "vstar_b200.h"

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxBeams = VSB_BEAM_MAX;
constexpr int kCap = 2048;                     // candidates at or above the threshold sorted in shared memory

template <bool F16>
__device__ __forceinline__ float round_dt(float x) {
  return F16 ? __half2float(__float2half_rn(x)) : __bfloat162float(__float2bfloat16_rn(x));
}

template <bool F16>
__device__ __forceinline__ float round_dt_d(double x) {
  return F16 ? __half2float(__double2half(x)) : __bfloat162float(__double2bfloat16(x));
}

// order-preserving 32-bit key of an fp32 value; -0 is folded onto +0 (they compare equal)
__device__ __forceinline__ uint32_t f32_key(float s) {
  uint32_t b = __float_as_uint(s);
  if (b == 0x80000000u) b = 0;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float key_f32(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key);
}

__device__ __forceinline__ float block_max_f(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct RowStats {
  float mx[kMaxBeams];
  double lse[kMaxBeams];
  float score[kMaxBeams];
  const float* row[kMaxBeams];
};

template <bool F16>
__device__ __forceinline__ uint32_t cand_key(const RowStats& st, int j, int i) {
  const float x = round_dt<F16>(st.row[j][i]);
  const float lp = round_dt_d<F16>((double)x - (double)st.mx[j] - st.lse[j]);
  return f32_key(lp + st.score[j]);
}

// sort cand[0, n) descending (bitonic over the next power of two, padded with 0 = below every real entry)
__device__ void sort_desc(unsigned long long* cand, int n) {
  const int t = threadIdx.x;
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = n + t; i < P; i += kThreads) cand[i] = 0ull;
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < (P >> 1); i += kThreads) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const unsigned long long a = cand[lo], b = cand[hi];
        if ((a < b) == desc) {
          cand[lo] = b;
          cand[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

template <bool F16>
__global__ void __launch_bounds__(kThreads, 1) beam_candidates_kernel(const float* __restrict__ logits, long long ld, int V, int k_in,
                                                                      int need, const int* __restrict__ rows,
                                                                      const float* __restrict__ scores, float* __restrict__ out_s,
                                                                      int* __restrict__ out_t, int* __restrict__ out_b) {
  __shared__ RowStats st;
  __shared__ unsigned long long cand[kCap];     // (key << 32) | ~flat: descending order = score desc, flat index asc
  __shared__ int hist[256];
  __shared__ int wsum[kWarps];
  __shared__ float redf[kWarps];
  __shared__ double redd[kWarps];
  __shared__ int s_bin, s_above, s_count;

  const int t = threadIdx.x, lane = t & 31;
  const int r = blockIdx.x;

  // ---- per row: max and log-sum-exp of the dtype-rounded logits
  for (int j = 0; j < k_in; ++j) {
    const float* row = logits + (long long)rows[r * k_in + j] * ld;
    float mx = -INFINITY;
    for (int i = t; i < V; i += kThreads) mx = fmaxf(mx, round_dt<F16>(row[i]));
    mx = block_max_f(mx, redf);
    double s = 0.0;
    for (int i = t; i < V; i += kThreads) s += (double)expf(round_dt<F16>(row[i]) - mx);
    s = block_sum_d(s, redd);
    if (t == 0) {
      st.row[j] = row;
      st.mx[j] = mx;
      st.lse[j] = log(s);
      st.score[j] = scores[r * k_in + j];
    }
  }
  __syncthreads();

  // ---- radix select of the need-th largest key (with multiplicity)
  uint32_t prefix = 0, mask = 0;
  int want = need;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if (t < 256) hist[t] = 0;
    __syncthreads();
    for (int j = 0; j < k_in; ++j) {
      for (int i0 = 0; i0 < V; i0 += kThreads) {
        const int i = i0 + t;
        int bin = -1;
        if (i < V) {
          const uint32_t key = cand_key<F16>(st, j, i);
          if ((key & mask) == prefix) bin = (int)((key >> shift) & 255u);
        }
        const unsigned grp = __match_any_sync(0xffffffffu, bin);            // one shared atomic per distinct bin of the warp
        if (bin >= 0 && lane == __ffs(grp) - 1) atomicAdd(&hist[bin], __popc(grp));
      }
    }
    __syncthreads();
    radix_bucket(hist, want, wsum, &s_bin, &s_above);
    prefix |= (uint32_t)s_bin << shift;
    mask |= 0xFFu << shift;
    want -= s_above;
  }
  const uint32_t tau = prefix;
  const int above = need - want;                                            // candidates with key > tau
  const int ncand = above + hist[s_bin];                                    // ... and with key >= tau
  if (t == 0) s_count = 0;
  __syncthreads();

  const bool wide = ncand > kCap;
  for (int j = 0; j < k_in; ++j) {
    for (int i = t; i < V; i += kThreads) {
      const uint32_t key = cand_key<F16>(st, j, i);
      if (key > tau || (!wide && key == tau))
        cand[atomicAdd(&s_count, 1)] = ((unsigned long long)key << 32) | (uint32_t)~(uint32_t)(j * V + i);
    }
  }
  __syncthreads();
  int n = ncand;
  if (wide) {
    // the `want` ties at tau with the lowest flattened indices, by one ordered pass
    int seen = 0;
    for (int f0 = 0; f0 < k_in * V && seen < want; f0 += kThreads) {
      const int f = f0 + t;
      const int j = f / V;
      const bool hit = f < k_in * V && cand_key<F16>(st, j, f - j * V) == tau;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) wsum[t >> 5] = __popc(bal);
      __syncthreads();
      int before = seen, total = 0;
      for (int q = 0; q < kWarps; ++q) {
        if (q < (t >> 5)) before += wsum[q];
        total += wsum[q];
      }
      const int pos = before + __popc(bal & ((1u << lane) - 1u));
      if (hit && pos < want) cand[above + pos] = ((unsigned long long)tau << 32) | (uint32_t)~(uint32_t)f;
      seen += total;
      __syncthreads();
    }
    n = need;
  }
  sort_desc(cand, n);
  if (t < need) {
    const unsigned long long c = cand[t];
    const int f = (int)~(uint32_t)c;
    out_s[r * need + t] = key_f32((uint32_t)(c >> 32));
    out_b[r * need + t] = f / V;
    out_t[r * need + t] = f - (f / V) * V;
  }
}

// one row range for every pair (vsb_copy_cache_rows_b16)
struct UniformPairs {
  int src[VSB_COPY_ROWS_MAX_PAIRS];
  int dst[VSB_COPY_ROWS_MAX_PAIRS];
  int lo, hi;
  __device__ __forceinline__ int lo_of(int) const { return lo; }
  __device__ __forceinline__ int hi_of(int) const { return hi; }
};

// a row range per pair (vsb_copy_slot_rows_b16); 16-bit slots keep the parameters inside the 4 KB kernel-argument limit
struct RangedPairs {
  unsigned short src[VSB_COPY_ROWS_MAX_PAIRS];
  unsigned short dst[VSB_COPY_ROWS_MAX_PAIRS];
  int lo[VSB_COPY_ROWS_MAX_PAIRS];
  int hi[VSB_COPY_ROWS_MAX_PAIRS];
  __device__ __forceinline__ int lo_of(int p) const { return lo[p]; }
  __device__ __forceinline__ int hi_of(int p) const { return hi[p]; }
};

// grid (chunks, layers, pairs): rows [lo, hi) of one slot of one layer, as VEC-element vectors
template <typename VEC, typename PAIRS>
__global__ void __launch_bounds__(256) copy_cache_rows_kernel(unsigned short* cache, long long layer_stride, long long slot_stride,
                                                              long long row_stride, int row_elems, const PAIRS pairs) {
  constexpr int kVec = sizeof(VEC) / 2;
  const int p = blockIdx.z;
  const int lo = pairs.lo_of(p), hi = pairs.hi_of(p);
  unsigned short* base = cache + (long long)blockIdx.y * layer_stride;
  const VEC* src = reinterpret_cast<const VEC*>(base + (long long)pairs.src[p] * slot_stride);
  VEC* dst = reinterpret_cast<VEC*>(base + (long long)pairs.dst[p] * slot_stride);
  const int per_row = row_elems / kVec;
  const long long rs = row_stride / kVec;
  const long long total = (long long)(hi - lo) * per_row;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = lo + e / per_row, c = e % per_row;
    dst[row * rs + c] = src[row * rs + c];
  }
}

// one launch for npairs pairs of at most `rows` rows each
template <typename PAIRS>
void launch_copy_rows(void* cache, int layers, long long layer_stride, long long slot_stride, long long row_stride, int row_elems,
                      const PAIRS& pp, int npairs, int rows, void* stream) {
  const bool vec = ((reinterpret_cast<uintptr_t>(cache) | (uintptr_t)layer_stride * 2 | (uintptr_t)slot_stride * 2 |
                     (uintptr_t)row_stride * 2 | (uintptr_t)row_elems * 2) & 15) == 0;
  const long long elems = (long long)rows * row_elems / (vec ? 8 : 1);
  const int chunks = (int)std::min<long long>((elems + 255) / 256, 64);
  dim3 grid(chunks, layers, npairs);
  if (vec)
    copy_cache_rows_kernel<uint4, PAIRS><<<grid, 256, 0, STREAM(stream)>>>((unsigned short*)cache, layer_stride, slot_stride, row_stride,
                                                                          row_elems, pp);
  else
    copy_cache_rows_kernel<unsigned short, PAIRS><<<grid, 256, 0, STREAM(stream)>>>((unsigned short*)cache, layer_stride, slot_stride,
                                                                                   row_stride, row_elems, pp);
}

// where the paged copy finds rows: the destination always in the pool through the page table, the source there too (FROM_POOL) or
// in a contiguous cache [layers][slots][rows][...]
struct PageRows {
  unsigned short* pool;
  long long layer_stride, page_stride, row_stride;
  const int* page_table;
  int pt_ld, page_shift;
  const unsigned short* src;
  long long src_layer_stride, src_slot_stride, src_row_stride;
  __device__ __forceinline__ long long pool_row(int slot, long long row) const {
    return (long long)__ldg(page_table + (long long)slot * pt_ld + (row >> page_shift)) * page_stride +
           (row & ((1 << page_shift) - 1)) * row_stride;
  }
};

// grid (chunks, layers, pairs): rows [lo, hi) of one page-table row of one layer, as VEC-element vectors
template <typename VEC, bool FROM_POOL>
__global__ void __launch_bounds__(256) copy_page_rows_kernel(const PageRows g, int row_elems, const RangedPairs pairs) {
  constexpr int kVec = sizeof(VEC) / 2;
  const int p = blockIdx.z;
  const int lo = pairs.lo[p], hi = pairs.hi[p];
  const int per_row = row_elems / kVec;
  const long long total = (long long)(hi - lo) * per_row;
  unsigned short* dbase = g.pool + (long long)blockIdx.y * g.layer_stride;
  const unsigned short* sbase = FROM_POOL ? dbase : g.src + (long long)blockIdx.y * g.src_layer_stride + (long long)pairs.src[p] * g.src_slot_stride;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = lo + e / per_row, c = e % per_row;
    const long long so = FROM_POOL ? g.pool_row(pairs.src[p], row) : row * g.src_row_stride;
    reinterpret_cast<VEC*>(dbase + g.pool_row(pairs.dst[p], row))[c] = reinterpret_cast<const VEC*>(sbase + so)[c];
  }
}

template <bool FROM_POOL>
void launch_copy_page_rows(const PageRows& g, int row_elems, const RangedPairs& pp, int layers, int npairs, int rows, void* stream) {
  const bool vec = ((reinterpret_cast<uintptr_t>(g.pool) | (uintptr_t)g.layer_stride * 2 | (uintptr_t)g.page_stride * 2 |
                     (uintptr_t)g.row_stride * 2 | (uintptr_t)row_elems * 2 |
                     (FROM_POOL ? 0 : (reinterpret_cast<uintptr_t>(g.src) | (uintptr_t)g.src_layer_stride * 2 | (uintptr_t)g.src_slot_stride * 2 |
                                       (uintptr_t)g.src_row_stride * 2))) & 15) == 0;
  const long long elems = (long long)rows * row_elems / (vec ? 8 : 1);
  const int chunks = (int)std::min<long long>((elems + 255) / 256, 64);
  dim3 grid(chunks, layers, npairs);
  if (vec)
    copy_page_rows_kernel<uint4, FROM_POOL><<<grid, 256, 0, STREAM(stream)>>>(g, row_elems, pp);
  else
    copy_page_rows_kernel<unsigned short, FROM_POOL><<<grid, 256, 0, STREAM(stream)>>>(g, row_elems, pp);
}

// (pool page, host slot) pairs of one launch: 8 bytes each keep the parameters inside the 4 KB kernel-argument limit
struct SwapPairs {
  int page[VSB_SWAP_PAGES_PER_LAUNCH];
  int slot[VSB_SWAP_PAGES_PER_LAUNCH];
};

struct SwapArea {
  uint4* pool;
  uint4* host;
  long long layer_stride, page_stride, slot_stride, host_layer_stride, vecs;    // in 16-byte vectors
};

// grid (chunks, layers, pairs): one page of one layer, 4 vectors in flight per thread (the host side is a PCIe round trip)
template <bool TO_HOST>
__global__ void __launch_bounds__(256) swap_pages_kernel(const SwapArea a, const SwapPairs pp) {
  constexpr int kUnroll = 4;
  const int p = blockIdx.z;
  const uint4* pool = a.pool + blockIdx.y * a.layer_stride + pp.page[p] * a.page_stride;
  const uint4* host = a.host + pp.slot[p] * a.slot_stride + blockIdx.y * a.host_layer_stride;
  const uint4* src = TO_HOST ? pool : host;
  uint4* dst = const_cast<uint4*>(TO_HOST ? host : pool);
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < a.vecs; e += kUnroll * step) {
    uint4 v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (e + u * step < a.vecs) v[u] = src[e + u * step];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (e + u * step < a.vecs) dst[e + u * step] = v[u];
  }
}

}  // namespace

extern "C" int vsb_beam_candidates_f32(const void* logits, long long ld, int V, int requests, int k_in, int k, const void* rows_i32,
                                       const void* scores_f32, int logit_dtype, void* out_score_f32, void* out_token_i32,
                                       void* out_beam_i32, void* stream) {
  VSB_CHECK_ARG(logits && rows_i32 && scores_f32 && out_score_f32 && out_token_i32 && out_beam_i32, "vsb_beam_candidates_f32: null pointer");
  VSB_CHECK_ARG(V > 0 && ld >= V, "vsb_beam_candidates_f32: bad V / ld");
  VSB_CHECK_ARG(k >= 1 && k <= VSB_BEAM_MAX, "vsb_beam_candidates_f32: k must be in [1, %d], got %d", VSB_BEAM_MAX, k);
  VSB_CHECK_ARG(k_in >= 1 && k_in <= k, "vsb_beam_candidates_f32: k_in must be in [1, k], got %d", k_in);
  VSB_CHECK_ARG((long long)k_in * V >= 2 * k && (long long)k_in * V < (1ll << 31), "vsb_beam_candidates_f32: k_in * V must be in [2k, 2^31)");
  VSB_CHECK_ARG(logit_dtype == VSB_DTYPE_BF16 || logit_dtype == VSB_DTYPE_F16, "vsb_beam_candidates_f32: logit_dtype must be VSB_DTYPE_BF16 or VSB_DTYPE_F16");
  if (requests <= 0) return VSB_OK;
  if (logit_dtype == VSB_DTYPE_F16)
    beam_candidates_kernel<true><<<requests, kThreads, 0, STREAM(stream)>>>((const float*)logits, ld, V, k_in, 2 * k, (const int*)rows_i32,
                                                                            (const float*)scores_f32, (float*)out_score_f32,
                                                                            (int*)out_token_i32, (int*)out_beam_i32);
  else
    beam_candidates_kernel<false><<<requests, kThreads, 0, STREAM(stream)>>>((const float*)logits, ld, V, k_in, 2 * k, (const int*)rows_i32,
                                                                             (const float*)scores_f32, (float*)out_score_f32,
                                                                             (int*)out_token_i32, (int*)out_beam_i32);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_copy_cache_rows_b16(void* cache, int layers, long long layer_stride, int slots, long long slot_stride, long long row_stride,
                                       int row_elems, const int* pairs_i32, int npairs, int lo, int hi, void* stream) {
  VSB_CHECK_ARG(cache && layers > 0 && slots > 0 && row_elems > 0 && row_stride >= row_elems, "vsb_copy_cache_rows_b16: bad args");
  VSB_CHECK_ARG(npairs >= 0 && npairs <= VSB_COPY_ROWS_MAX_PAIRS, "vsb_copy_cache_rows_b16: npairs must be in [0, %d], got %d",
                VSB_COPY_ROWS_MAX_PAIRS, npairs);
  VSB_CHECK_ARG(0 <= lo && lo <= hi && (long long)hi * row_stride <= slot_stride, "vsb_copy_cache_rows_b16: bad row range [%d, %d)", lo, hi);
  VSB_CHECK_ARG(npairs == 0 || pairs_i32, "vsb_copy_cache_rows_b16: null pair list");
  UniformPairs pp;
  for (int p = 0; p < npairs; ++p) {
    const int s = pairs_i32[2 * p], d = pairs_i32[2 * p + 1];
    VSB_CHECK_ARG(s >= 0 && s < slots && d >= 0 && d < slots, "vsb_copy_cache_rows_b16: pair %d (%d -> %d) outside [0, %d)", p, s, d, slots);
    for (int q = 0; q < npairs; ++q) {
      VSB_CHECK_ARG(pairs_i32[2 * q + 1] != s, "vsb_copy_cache_rows_b16: slot %d is both a source and a destination", s);
      VSB_CHECK_ARG(q == p || pairs_i32[2 * q + 1] != d, "vsb_copy_cache_rows_b16: slot %d is the destination of two pairs", d);
    }
    pp.src[p] = s;
    pp.dst[p] = d;
  }
  pp.lo = lo;
  pp.hi = hi;
  if (npairs == 0 || hi == lo) return VSB_OK;
  launch_copy_rows(cache, layers, layer_stride, slot_stride, row_stride, row_elems, pp, npairs, hi - lo, stream);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_copy_slot_rows_b16(void* cache, int layers, long long layer_stride, int slots, long long slot_stride, long long row_stride,
                                      int row_elems, const int* quads_i32, int npairs, void* stream) {
  VSB_CHECK_ARG(cache && layers > 0 && slots > 0 && slots <= 65536 && row_elems > 0 && row_stride >= row_elems,
                "vsb_copy_slot_rows_b16: bad args");
  VSB_CHECK_ARG(npairs >= 0 && npairs <= VSB_COPY_ROWS_MAX_PAIRS, "vsb_copy_slot_rows_b16: npairs must be in [0, %d], got %d",
                VSB_COPY_ROWS_MAX_PAIRS, npairs);
  VSB_CHECK_ARG(npairs == 0 || quads_i32, "vsb_copy_slot_rows_b16: null pair list");
  RangedPairs pp;
  int rows = 0;
  for (int p = 0; p < npairs; ++p) {
    const int s = quads_i32[4 * p], d = quads_i32[4 * p + 1], lo = quads_i32[4 * p + 2], hi = quads_i32[4 * p + 3];
    VSB_CHECK_ARG(s >= 0 && s < slots && d >= 0 && d < slots, "vsb_copy_slot_rows_b16: pair %d (%d -> %d) outside [0, %d)", p, s, d, slots);
    VSB_CHECK_ARG(0 <= lo && lo <= hi && (long long)hi * row_stride <= slot_stride, "vsb_copy_slot_rows_b16: pair %d: bad row range [%d, %d)",
                  p, lo, hi);
    for (int q = 0; q < npairs; ++q) {
      VSB_CHECK_ARG(quads_i32[4 * q + 1] != s, "vsb_copy_slot_rows_b16: slot %d is both a source and a destination", s);
      VSB_CHECK_ARG(q == p || quads_i32[4 * q + 1] != d, "vsb_copy_slot_rows_b16: slot %d is the destination of two pairs", d);
    }
    pp.src[p] = (unsigned short)s;
    pp.dst[p] = (unsigned short)d;
    pp.lo[p] = lo;
    pp.hi[p] = hi;
    rows = std::max(rows, hi - lo);
  }
  if (npairs == 0 || rows == 0) return VSB_OK;
  launch_copy_rows(cache, layers, layer_stride, slot_stride, row_stride, row_elems, pp, npairs, rows, stream);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_copy_page_rows_b16(void* pool, int layers, long long layer_stride, long long page_stride, int page_rows, long long row_stride,
                                      int row_elems, const void* page_table_i32, int pt_ld, int slots, const void* src, long long src_layer_stride,
                                      long long src_slot_stride, long long src_row_stride, int src_slots, const int* quads_i32, int npairs,
                                      void* stream) {
  VSB_CHECK_ARG(pool && page_table_i32 && layers > 0 && slots > 0 && slots <= 65536 && pt_ld > 0 && row_elems > 0 && row_stride >= row_elems &&
                    page_stride >= (long long)page_rows * row_stride,
                "vsb_copy_page_rows_b16: bad args");
  VSB_CHECK_ARG(page_rows >= 16 && (page_rows & (page_rows - 1)) == 0, "vsb_copy_page_rows_b16: page_rows %d is not a power of two >= 16",
                page_rows);
  VSB_CHECK_ARG(src == nullptr || (src_slots > 0 && src_slots <= 65536 && src_row_stride >= row_elems),
                "vsb_copy_page_rows_b16: bad contiguous source");
  VSB_CHECK_ARG(npairs >= 0 && npairs <= VSB_COPY_ROWS_MAX_PAIRS, "vsb_copy_page_rows_b16: npairs must be in [0, %d], got %d",
                VSB_COPY_ROWS_MAX_PAIRS, npairs);
  VSB_CHECK_ARG(npairs == 0 || quads_i32, "vsb_copy_page_rows_b16: null pair list");
  const long long row_cap = (long long)pt_ld * page_rows;
  RangedPairs pp;
  int rows = 0;
  for (int p = 0; p < npairs; ++p) {
    const int s = quads_i32[4 * p], d = quads_i32[4 * p + 1], lo = quads_i32[4 * p + 2], hi = quads_i32[4 * p + 3];
    VSB_CHECK_ARG(s >= 0 && s < (src ? src_slots : slots) && d >= 0 && d < slots, "vsb_copy_page_rows_b16: pair %d (%d -> %d) outside the tables",
                  p, s, d);
    VSB_CHECK_ARG(0 <= lo && lo <= hi && hi <= row_cap && (src == nullptr || (long long)hi * src_row_stride <= src_slot_stride),
                  "vsb_copy_page_rows_b16: pair %d: bad row range [%d, %d)", p, lo, hi);
    for (int q = 0; q < npairs; ++q) {
      VSB_CHECK_ARG(src || quads_i32[4 * q + 1] != s, "vsb_copy_page_rows_b16: row %d is both a source and a destination", s);
      VSB_CHECK_ARG(q == p || quads_i32[4 * q + 1] != d, "vsb_copy_page_rows_b16: row %d is the destination of two pairs", d);
    }
    pp.src[p] = (unsigned short)s;
    pp.dst[p] = (unsigned short)d;
    pp.lo[p] = lo;
    pp.hi[p] = hi;
    rows = std::max(rows, hi - lo);
  }
  if (npairs == 0 || rows == 0) return VSB_OK;
  PageRows g;
  g.pool = (unsigned short*)pool;
  g.layer_stride = layer_stride; g.page_stride = page_stride; g.row_stride = row_stride;
  g.page_table = (const int*)page_table_i32;
  g.pt_ld = pt_ld;
  g.page_shift = __builtin_ctz((unsigned)page_rows);
  g.src = (const unsigned short*)src;
  g.src_layer_stride = src_layer_stride; g.src_slot_stride = src_slot_stride; g.src_row_stride = src_row_stride;
  if (src)
    launch_copy_page_rows<false>(g, row_elems, pp, layers, npairs, rows, stream);
  else
    launch_copy_page_rows<true>(g, row_elems, pp, layers, npairs, rows, stream);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_swap_pages_b16(void* pool, int layers, long long layer_stride, int n_pages, long long page_stride, long long page_elems,
                                  void* host, int host_slots, long long host_slot_stride, long long host_layer_stride, const int* pages_i32,
                                  const int* slots_i32, int n, int to_host, void* stream) {
  VSB_CHECK_ARG(pool && host, "vsb_swap_pages_b16: null pointer");
  VSB_CHECK_ARG(n >= 0 && (n == 0 || (pages_i32 && slots_i32)), "vsb_swap_pages_b16: null page list or n < 0");
  VSB_CHECK_ARG(layers > 0 && n_pages > 0 && host_slots > 0 && page_elems > 0 && page_stride >= page_elems &&
                    layer_stride >= (long long)n_pages * page_stride && host_layer_stride >= page_elems &&
                    host_slot_stride >= (long long)layers * host_layer_stride,
                "vsb_swap_pages_b16: bad shape");
  VSB_CHECK_ARG(((reinterpret_cast<uintptr_t>(pool) | reinterpret_cast<uintptr_t>(host) | (uintptr_t)(layer_stride * 2) |
                  (uintptr_t)(page_stride * 2) | (uintptr_t)(page_elems * 2) | (uintptr_t)(host_slot_stride * 2) |
                  (uintptr_t)(host_layer_stride * 2)) & 15) == 0,
                "vsb_swap_pages_b16: pointers and strides must be 16-byte aligned");
  std::vector<int> seen((size_t)(to_host ? host_slots : n_pages), 0);
  for (int i = 0; i < n; ++i) {
    const int pg = pages_i32[i], sl = slots_i32[i];
    VSB_CHECK_ARG(pg >= 0 && pg < n_pages, "vsb_swap_pages_b16: pair %d: page %d outside [0, %d)", i, pg, n_pages);
    VSB_CHECK_ARG(sl >= 0 && sl < host_slots, "vsb_swap_pages_b16: pair %d: host slot %d outside [0, %d)", i, sl, host_slots);
    int& d = seen[to_host ? sl : pg];
    VSB_CHECK_ARG(!d, "vsb_swap_pages_b16: %s %d is the destination of two pairs", to_host ? "host slot" : "page", to_host ? sl : pg);
    d = 1;
  }
  void* mapped = nullptr;
  if (cudaHostGetDevicePointer(&mapped, host, 0) != cudaSuccess || mapped == nullptr) {
    cudaGetLastError();
    VSB_CHECK_ARG(false, "vsb_swap_pages_b16: the swap area is not mapped pinned host memory");
  }
  if (n == 0) return VSB_OK;
  SwapArea a;
  a.pool = (uint4*)pool;
  a.host = (uint4*)mapped;
  a.layer_stride = layer_stride / 8; a.page_stride = page_stride / 8;
  a.slot_stride = host_slot_stride / 8; a.host_layer_stride = host_layer_stride / 8;
  a.vecs = page_elems / 8;
  const int chunks = (int)std::min<long long>((a.vecs + 1023) / 1024, 64);
  for (int i = 0; i < n; i += VSB_SWAP_PAGES_PER_LAUNCH) {
    const int m = std::min(n - i, VSB_SWAP_PAGES_PER_LAUNCH);
    SwapPairs pp;
    std::copy(pages_i32 + i, pages_i32 + i + m, pp.page);
    std::copy(slots_i32 + i, slots_i32 + i + m, pp.slot);
    dim3 grid(chunks, layers, m);
    if (to_host)
      swap_pages_kernel<true><<<grid, 256, 0, STREAM(stream)>>>(a, pp);
    else
      swap_pages_kernel<false><<<grid, 256, 0, STREAM(stream)>>>(a, pp);
    VSB_LAUNCH_CHECK();
  }
  return VSB_OK;
}
