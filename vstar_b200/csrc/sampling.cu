// Sampled decoding of the SEAL VQA LLM: one CTA per row of fp32 logits draws one token with the semantics of HF `sample()`
// (TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> multinomial(softmax)), with the logits rounded to the
// engine dtype first as the reference's fp16 lm_head output is.  oracle/sampling_oracle.py restates every step.
//
// Per row:
//   1. v_i = dtype(float(dtype(x_i)) / T).  v is a 16-bit value, so it is carried as a 16-bit order-preserving key.
//   2. top-k: the key of the k-th largest v (with multiplicity) by a two-pass 8+8 bit radix select; every v >= it is kept,
//      so ties at the k-th value all survive.
//   3. probabilities e_i = exp(v_i - max) in fp64 (1 for the max itself); top-p keeps descending position j while the mass at
//      or after j exceeds (1 - top_p) of the total (HF's ascending cumsum rule; position 0 always kept).
//   4. inverse CDF at u = Philox4x32-10(key = seed, counter = (step, 0, 0, 0)) -> 53-bit uniform, over the kept tokens in
//      descending v, ties by ascending token id.
// vsb_sample_rows_f32 takes one temperature / top_k / top_p / step for every row; vsb_sample_rows_var_f32 (the decode stream)
// reads them per row from device arrays.  Both run the same kernel template, so a row draws the same token through either.
// Fast path (<= kCap candidates, every default top_k = 50 row that is not a wide tie): compact the candidates into shared
// memory, bitonic-sort them, scan their masses.  Otherwise (no top-k on a row wider than kCap, or a tie wider than kCap at the
// k-th value): binary searches over the row's keys, each probe one block-reduced pass over the row; tokens of one key share one
// probability, so the position inside the chosen key is found arithmetically and then by one ordered pass.
#include "common.cuh"
#include "radix_select.cuh"
#include "vstar_b200.h"

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kCap = 2048;

__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0;
    c[1] = lo1;
    c[2] = n2;
    c[3] = lo0;
  }
}

// order-preserving 16-bit key of dtype(float(dtype(x)) / T); -0 is folded onto +0 (they compare equal)
template <bool F16>
__device__ __forceinline__ uint32_t logit_key(float x, float T) {
  uint32_t b;
  if (F16) {
    b = __half_as_ushort(__float2half_rn(__half2float(__float2half_rn(x)) / T));
  } else {
    b = __bfloat16_as_ushort(__float2bfloat16_rn(__bfloat162float(__float2bfloat16_rn(x)) / T));
  }
  if (b == 0x8000u) b = 0;
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}

template <bool F16>
__device__ __forceinline__ float key_value(uint32_t key) {
  const unsigned short b = (key & 0x8000u) ? (unsigned short)(key & 0x7FFFu) : (unsigned short)(~key & 0xFFFFu);
  return F16 ? __half2float(__ushort_as_half(b)) : __bfloat162float(__ushort_as_bfloat16(b));
}

// unnormalised probability of a key: exp(v - max) in fp64, exactly 1 for the max (also when the max is +-inf)
template <bool F16>
__device__ __forceinline__ double key_mass(uint32_t key, uint32_t kmax, double m) {
  return key == kmax ? 1.0 : exp((double)key_value<F16>(key) - m);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum_d(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = warp_sum_d(lane < kWarps ? red[lane] : 0.0);
  return v;
}

template <bool F16>
__device__ __forceinline__ double mass_ge(const float* row, int n, float T, uint32_t lo, uint32_t kmax, double m, double* red) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const uint32_t key = logit_key<F16>(row[i], T);
    if (key >= lo) s += key_mass<F16>(key, kmax, m);
  }
  return block_sum_d(s, red);
}

template <bool F16>
__device__ __forceinline__ int count_eq(const float* row, int n, float T, uint32_t key0) {
  int c = 0;
  for (int i = threadIdx.x; i < n; i += kThreads) c += logit_key<F16>(row[i], T) == key0;
  c = __reduce_add_sync(0xffffffffu, c);
  __shared__ int total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicAdd(&total, c);
  __syncthreads();
  const int r = total;
  __syncthreads();
  return r;
}

// PER_ROW: temperature, top_k, top_p and step come from the row's entry of the device arrays (a decode stream, every request at
// its own step with its own settings); otherwise from the scalar arguments, and the arrays are not read.
template <bool F16, bool PER_ROW>
__global__ void __launch_bounds__(kThreads, 1) sample_rows_kernel(const float* __restrict__ logits, long long ld, int n, float T, int top_k,
                                                               float top_p, const long long* __restrict__ seeds, int step,
                                                               const float* __restrict__ T_row, const int* __restrict__ top_k_row,
                                                               const float* __restrict__ top_p_row, const int* __restrict__ step_row,
                                                               int* __restrict__ out) {
  __shared__ unsigned long long cand[kCap];              // (key << 32) | ~id: descending order = v desc, id asc
  __shared__ double cum[kCap];
  __shared__ int hist[256];
  __shared__ int wsum[kWarps];
  __shared__ double red[kWarps];
  __shared__ int s_bin, s_above, s_count;
  __shared__ unsigned int s_kmax, s_kmin;
  __shared__ double s_u;

  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const float* row = logits + (long long)blockIdx.x * ld;
  if (PER_ROW) {
    T = T_row[blockIdx.x];
    top_k = top_k_row[blockIdx.x];
    top_p = top_p_row[blockIdx.x];
    step = step_row[blockIdx.x];
  }
  if (t == 0) {
    const unsigned long long seed = (unsigned long long)seeds[blockIdx.x];
    uint32_t c[4] = {(uint32_t)step, 0u, 0u, 0u};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    s_u = ((double)(c[0] >> 5) * 67108864.0 + (double)(c[1] >> 6)) * (1.0 / 9007199254740992.0);   // [0, 1), 53 bits
    s_kmax = 0;
    s_kmin = 0xFFFFu;
    s_count = 0;
  }
  if (t < 256) hist[t] = 0;
  __syncthreads();

  // ---- pass 1: max and min key, histogram of the high byte
  const bool topk = top_k > 0 && top_k < n;
  unsigned int mx = 0, mn = 0xFFFFu;
  for (int i = t; i < n; i += kThreads) {
    const uint32_t key = logit_key<F16>(row[i], T);
    mx = max(mx, key);
    mn = min(mn, key);
    if (topk) atomicAdd(&hist[key >> 8], 1);
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  mn = __reduce_min_sync(0xffffffffu, mn);
  if (lane == 0) {
    atomicMax(&s_kmax, mx);
    atomicMin(&s_kmin, mn);
  }
  __syncthreads();
  const uint32_t kmax = s_kmax;
  const double m = (double)key_value<F16>(kmax);

  // ---- top-k threshold key (ties at the k-th value kept; without top-k the smallest key, so it is a key of the row)
  uint32_t ktau = s_kmin;
  int ncand = n;
  if (topk) {
    radix_bucket(hist, top_k, wsum, &s_bin, &s_above);
    const uint32_t hb = (uint32_t)s_bin;
    const int above = s_above;
    if (t < 256) hist[t] = 0;
    __syncthreads();
    for (int i = t; i < n; i += kThreads) {
      const uint32_t key = logit_key<F16>(row[i], T);
      if ((key >> 8) == hb) atomicAdd(&hist[key & 255u], 1);
    }
    __syncthreads();
    radix_bucket(hist, top_k - above, wsum, &s_bin, &s_above);
    ktau = (hb << 8) | (uint32_t)s_bin;
    ncand = above + s_above + hist[s_bin];
  }
  const bool nucleus = top_p < 1.f;
  const double thr = 1.0 - (double)top_p;               // remove while the mass at and after a position is <= thr
  const double u = s_u;

  if (ncand <= kCap) {
    // ---- fast path: compact, sort, scan
    for (int i = t; i < n; i += kThreads) {
      const uint32_t key = logit_key<F16>(row[i], T);
      if (key >= ktau) cand[atomicAdd(&s_count, 1)] = ((unsigned long long)key << 32) | (uint32_t)~(uint32_t)i;
    }
    int P = 1;
    while (P < ncand) P <<= 1;
    __syncthreads();
    for (int i = ncand + t; i < P; i += kThreads) cand[i] = 0ull;
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
    // inclusive scan of the masses: thread t owns positions 2t, 2t+1
    const int j0 = 2 * t;
    const double a0 = j0 < ncand ? key_mass<F16>((uint32_t)(cand[j0] >> 32), kmax, m) : 0.0;
    const double a1 = j0 + 1 < ncand ? key_mass<F16>((uint32_t)(cand[j0 + 1] >> 32), kmax, m) : 0.0;
    double s = a0 + a1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane == 31) red[w] = s;
    __syncthreads();
    double off = 0.0;
    for (int i = 0; i < w; ++i) off += red[i];
    const double excl = off + s - (a0 + a1);
    if (j0 < kCap) cum[j0] = excl + a0;
    if (j0 + 1 < kCap) cum[j0 + 1] = excl + a0 + a1;
    if (t == 0) s_count = 0;
    __syncthreads();
    const double E = cum[ncand - 1];
    int J = ncand;
    if (nucleus) {
      const double lim = thr * E;
      int keep = 0;
      for (int j = t; j < ncand; j += kThreads) keep += (E - (j ? cum[j - 1] : 0.0)) > lim;
      keep = __reduce_add_sync(0xffffffffu, keep);
      if (lane == 0) atomicAdd(&s_count, keep);
      __syncthreads();
      J = max(s_count, 1);
      __syncthreads();
      if (t == 0) s_count = 0;
      __syncthreads();
    }
    const double target = u * cum[J - 1];
    int below = 0;
    for (int j = t; j < J; j += kThreads) below += cum[j] <= target;
    below = __reduce_add_sync(0xffffffffu, below);
    if (lane == 0) atomicAdd(&s_count, below);
    __syncthreads();
    if (t == 0) out[blockIdx.x] = (int)~(uint32_t)cand[min(s_count, J - 1)];
    return;
  }

  // ---- wide path: binary searches over keys in [ktau, kmax]
  const double E = mass_ge<F16>(row, n, T, ktau, kmax, m, red);
  uint32_t kb = ktau;                                    // lowest kept key
  int rb;                                                // tokens of key kb kept (the first rb by ascending id)
  if (nucleus) {
    const double lim = thr * E;
    if (!(E > lim)) {                                   // top_p = 0: the largest token only
      kb = kmax;
      rb = 1;
    } else {                                            // smallest K with mass(keys <= K) > lim
      uint32_t lo = ktau, hi = kmax;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (E - mass_ge<F16>(row, n, T, mid + 1, kmax, m, red) > lim) hi = mid;
        else lo = mid + 1;
      }
      kb = lo;
      const int g = count_eq<F16>(row, n, T, kb);
      const double p = key_mass<F16>(kb, kmax, m);
      const double L = E - mass_ge<F16>(row, n, T, kb, kmax, m, red);   // mass strictly below kb
      const double x = p > 0.0 ? floor((lim - L) / p) : 0.0;
      rb = (int)max(1.0, min((double)g, (double)g - x));
    }
  } else {
    rb = count_eq<F16>(row, n, T, kb);
  }
  const double above_kb = mass_ge<F16>(row, n, T, kb + 1, kmax, m, red);
  const double Ek = above_kb + (double)rb * key_mass<F16>(kb, kmax, m);
  const double target = u * Ek;
  uint32_t lo = kb, hi = kmax;                           // smallest K >= kb with mass(keys > K) <= target
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (mass_ge<F16>(row, n, T, mid + 1, kmax, m, red) <= target) hi = mid;
    else lo = mid + 1;
  }
  const uint32_t K = lo;
  const double base = K == kb ? above_kb : mass_ge<F16>(row, n, T, K + 1, kmax, m, red);
  const int lim_r = K == kb ? rb : count_eq<F16>(row, n, T, K);
  const double pK = key_mass<F16>(K, kmax, m);
  const int r = pK > 0.0 ? (int)max(0.0, min((double)(lim_r - 1), floor((target - base) / pK))) : 0;
  // the r-th token of key K by ascending id
  int seen = 0;
  for (int i0 = 0; i0 < n; i0 += kThreads) {
    const int i = i0 + t;
    const bool hit = i < n && logit_key<F16>(row[i], T) == K;
    const unsigned int bal = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    int before = seen, total = 0;
    for (int q = 0; q < kWarps; ++q) {
      if (q < w) before += wsum[q];
      total += wsum[q];
    }
    if (hit && before + __popc(bal & ((1u << lane) - 1u)) == r) out[blockIdx.x] = i;
    seen += total;
    __syncthreads();
    if (seen > r) break;
  }
}

template <bool PER_ROW>
void launch_sample_rows(const void* logits, long long ld, int rows, int n, float temperature, int top_k, float top_p, int logit_dtype,
                        const void* seeds, int step, const void* T_row, const void* top_k_row, const void* top_p_row,
                        const void* step_row, void* idx, void* stream) {
  if (logit_dtype == VSB_DTYPE_F16)
    sample_rows_kernel<true, PER_ROW><<<rows, kThreads, 0, STREAM(stream)>>>(
        (const float*)logits, ld, n, temperature, top_k, top_p, (const long long*)seeds, step, (const float*)T_row,
        (const int*)top_k_row, (const float*)top_p_row, (const int*)step_row, (int*)idx);
  else
    sample_rows_kernel<false, PER_ROW><<<rows, kThreads, 0, STREAM(stream)>>>(
        (const float*)logits, ld, n, temperature, top_k, top_p, (const long long*)seeds, step, (const float*)T_row,
        (const int*)top_k_row, (const float*)top_p_row, (const int*)step_row, (int*)idx);
}

}  // namespace

extern "C" int vsb_sample_rows_f32(const void* logits, long long ld, int rows, int n, float temperature, int top_k, float top_p,
                                   int logit_dtype, const void* seeds_i64, int step, void* idx_i32, void* stream) {
  VSB_CHECK_ARG(logits && seeds_i64 && idx_i32 && n > 0 && ld >= n, "vsb_sample_rows_f32: bad args");
  VSB_CHECK_ARG(temperature > 0.f, "vsb_sample_rows_f32: temperature must be > 0 (greedy decoding is vsb_argmax_rows_f32)");
  VSB_CHECK_ARG(top_k >= 0, "vsb_sample_rows_f32: top_k must be >= 0 (0 = no top-k filter)");
  VSB_CHECK_ARG(top_p >= 0.f && top_p <= 1.f, "vsb_sample_rows_f32: top_p must be in [0, 1] (1 = no nucleus filter)");
  VSB_CHECK_ARG(logit_dtype == VSB_DTYPE_BF16 || logit_dtype == VSB_DTYPE_F16, "vsb_sample_rows_f32: logit_dtype must be VSB_DTYPE_BF16 or VSB_DTYPE_F16");
  if (rows <= 0) return VSB_OK;
  launch_sample_rows<false>(logits, ld, rows, n, temperature, top_k, top_p, logit_dtype, seeds_i64, step, nullptr, nullptr, nullptr,
                            nullptr, idx_i32, stream);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_sample_rows_var_f32(const void* logits, long long ld, int rows, int n, const void* temperature_f32,
                                       const void* top_k_i32, const void* top_p_f32, int logit_dtype, const void* seeds_i64,
                                       const void* steps_i32, void* idx_i32, void* stream) {
  VSB_CHECK_ARG(logits && temperature_f32 && top_k_i32 && top_p_f32 && seeds_i64 && steps_i32 && idx_i32 && n > 0 && ld >= n,
                "vsb_sample_rows_var_f32: bad args");
  VSB_CHECK_ARG(logit_dtype == VSB_DTYPE_BF16 || logit_dtype == VSB_DTYPE_F16, "vsb_sample_rows_var_f32: logit_dtype must be VSB_DTYPE_BF16 or VSB_DTYPE_F16");
  if (rows <= 0) return VSB_OK;
  launch_sample_rows<true>(logits, ld, rows, n, 0.f, 0, 1.f, logit_dtype, seeds_i64, 0, temperature_f32, top_k_i32, top_p_f32, steps_i32,
                           idx_i32, stream);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}
