// Memory-bound row kernels of the VSM hot path: norms, RoPE, embedding splice,
// patchify (im2col), positional add, OWL token merge, small adds.
// All are HBM-bound streaming kernels: 16-byte vectorised, coalesced loads,
// warp-shuffle reductions, one row per warp/block, no shared-memory staging
// beyond the block reduction scratch.
#include "common.cuh"
#include "vstar_b200.h"

namespace {

// ------------------------------------------------------------------ LayerNorm / RMSNorm: ONE WARP PER ROW
// The whole row lives in the warp's registers (MAXV 16-byte vectors per lane), statistics by warp shuffles only - no
// shared memory, no __syncthreads - and every lane has MAXV independent 16 B loads in flight, which is what an HBM-bound
// row kernel needs (the previous block-per-row version sat at ~2.5 TB/s).
template <int MAXV, typename T>
__device__ __forceinline__ int load_row(const T* __restrict__ xr, int nvec, int lane, float (*v)[8]) {
  using E = ElemT<T>;
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint4 u = *reinterpret_cast<const uint4*>(xr + vi * 8);
      float2 t;
      t = E::unpack2(u.x); v[i][0] = t.x; v[i][1] = t.y;
      t = E::unpack2(u.y); v[i][2] = t.x; v[i][3] = t.y;
      t = E::unpack2(u.z); v[i][4] = t.x; v[i][5] = t.y;
      t = E::unpack2(u.w); v[i][6] = t.x; v[i][7] = t.y;
      ++cnt;
    }
  }
  return cnt;
}

template <typename T>
__device__ __forceinline__ void unpack8(const uint4 u, float* f) {
  using E = ElemT<T>;
  float2 t;
  t = E::unpack2(u.x); f[0] = t.x; f[1] = t.y;
  t = E::unpack2(u.y); f[2] = t.x; f[3] = t.y;
  t = E::unpack2(u.z); f[4] = t.x; f[5] = t.y;
  t = E::unpack2(u.w); f[6] = t.x; f[7] = t.y;
}
template <typename T>
__device__ __forceinline__ uint4 pack8(const float* o) {
  using E = ElemT<T>;
  uint4 u;
  u.x = E::pack2(o[0], o[1]); u.y = E::pack2(o[2], o[3]); u.z = E::pack2(o[4], o[5]); u.w = E::pack2(o[6], o[7]);
  return u;
}

// y = (x - mean) * rsqrt(var + eps) * w + b ; fp32 statistics (two-pass over registers), T (bf16 / f16) in/out, optional GELU
template <int MAXV, typename T>
__global__ void __launch_bounds__(128) layernorm_kernel(const T* __restrict__ x, long long ldx, const T* __restrict__ w,
                                                        const T* __restrict__ b, T* __restrict__ y, long long ldy,
                                                        int rows, int cols, float eps, int act) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + (long long)row * ldx;
  T* yr = y + (long long)row * ldy;
  const int nvec = cols >> 3;
  float v[MAXV][8];
  load_row<MAXV, T>(xr, nvec, lane, v);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  const float mean = warp_sum(s) / (float)cols;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float wf[8], bfv[8], o[8];
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(w + vi * 8)), wf);
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(b + vi * 8)), bfv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = (v[i][j] - mean) * rstd * wf[j] + bfv[j];
        if (act == VSB_EPI_GELU) o[j] = gelu_erf_f(o[j]);
      }
      *reinterpret_cast<uint4*>(yr + vi * 8) = pack8<T>(o);
    }
  }
}

// HF LlamaRMSNorm: y = w * T( x * rsqrt(mean(x^2) + eps) )     (transformers/models/llama/modeling_llama.py:53-67)
template <int MAXV, typename T>
__global__ void __launch_bounds__(128) rmsnorm_kernel(const T* __restrict__ x, long long ldx, const T* __restrict__ w,
                                                      T* __restrict__ y, long long ldy, int rows, int cols, float eps) {
  using E = ElemT<T>;
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + (long long)row * ldx;
  T* yr = y + (long long)row * ldy;
  const int nvec = cols >> 3;
  float v[MAXV][8];
  load_row<MAXV, T>(xr, nvec, lane, v);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) sq += v[i][j] * v[i][j];
    }
  const float rstd = rsqrtf(warp_sum(sq) / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float wf[8], o[8];
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(w + vi * 8)), wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = wf[j] * E::round(v[i][j] * rstd);
      *reinterpret_cast<uint4*>(yr + vi * 8) = pack8<T>(o);
    }
  }
}

// few rows (decode): one 256-thread block per row so the row's loads are all in flight at once; a single warp per row
// (above) serialises 16 dependent-latency loads.  Same arithmetic, same rounding.
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_row_kernel(const T* __restrict__ x, long long ldx, const T* __restrict__ w,
                                                          T* __restrict__ y, long long ldy, int cols, float eps) {
  using E = ElemT<T>;
  pdl_prologue();
  __shared__ float red[32];
  const T* xr = x + (long long)blockIdx.x * ldx;
  T* yr = y + (long long)blockIdx.x * ldy;
  const int nvec = cols >> 3;
  constexpr int MAXV = 4;                      // cols <= 8192
  float v[MAXV][8], wf[MAXV][8];
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = threadIdx.x + i * 256;
    if (vi < nvec) {
      unpack8<T>(*reinterpret_cast<const uint4*>(xr + vi * 8), v[i]);
      unpack8<T>(__ldg(reinterpret_cast<const uint4*>(w + vi * 8)), wf[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sq += v[i][j] * v[i][j];
    }
  }
  const float rstd = rsqrtf(block_sum(sq, red) / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = threadIdx.x + i * 256;
    if (vi < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = wf[i][j] * E::round(v[i][j] * rstd);
      *reinterpret_cast<uint4*>(yr + vi * 8) = pack8<T>(o);
    }
  }
}

// ------------------------------------------------------------------ RoPE (rotate-half), in place on q and k
// x' = T( T(x*cos) + T(rot(x)*sin) ); cos/sin come from host-built T tables [max_pos, D/2]
// (built with the same fp32 torch ops as HF: transformers/models/llama/modeling_llama.py:117-168),
// so the rotation is bit-identical to the reference's bf16 / fp16 path.  Row layout: [.., 3*H*D] = q | k | v.
// logical row r (0..rows) lives at physical row (r / T) * group_stride + group_offset + r % T (KV-cache layout
// [B, Tmax, 3*H*D]); its position = positions[r] if given else pos0 + (r % T)
template <typename E_T>
__global__ void rope_kernel(E_T* __restrict__ qkv, long long ld, int rows, int T, int H, int D, int pos0,
                            const E_T* __restrict__ cos_t, const E_T* __restrict__ sin_t, const int* __restrict__ positions,
                            long long group_stride, long long group_offset) {
  using E = ElemT<E_T>;
  pdl_prologue();
  const int row = blockIdx.x;
  if (row >= rows) return;
  const int pos = positions ? positions[row] : pos0 + (row % T);
  const int half = D >> 1;
  const int hv = half >> 3;                 // 16-byte vectors per half head
  E_T* base = qkv + ((long long)(row / T) * group_stride + group_offset + (row % T)) * ld;
  const E_T* cr = cos_t + (long long)pos * half;
  const E_T* sr = sin_t + (long long)pos * half;
  // one thread = 8 consecutive (i, i+half) pairs of one head of q or k
  for (int idx = threadIdx.x; idx < 2 * H * hv; idx += blockDim.x) {
    const int hh = idx / hv;                // 0..2H-1 : q heads then k heads (contiguous: k starts at H*D)
    const int v = idx - hh * hv;
    E_T* p = base + (long long)hh * D + v * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(p);
    const uint4 b = *reinterpret_cast<const uint4*>(p + half);
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(cr + v * 8));
    const uint4 s = __ldg(reinterpret_cast<const uint4*>(sr + v * 8));
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, cw[4] = {c.x, c.y, c.z, c.w}, sw[4] = {s.x, s.y, s.z, s.w};
    uint32_t oa[4], ob[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x1 = E::unpack2(aw[j]), x2 = E::unpack2(bw[j]), cs = E::unpack2(cw[j]), sn = E::unpack2(sw[j]);
      oa[j] = E::pack2(E::round(x1.x * cs.x) + E::round(-x2.x * sn.x), E::round(x1.y * cs.y) + E::round(-x2.y * sn.y));
      ob[j] = E::pack2(E::round(x2.x * cs.x) + E::round(x1.x * sn.x), E::round(x2.y * cs.y) + E::round(x1.y * sn.y));
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(p + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
  }
}

// RoPE + scatter of one fused q|k|v row per decode row into the KV cache: row b of qkv goes to cache row
// slot[b]*Tmax + len[b] with q and k rotated at position pos[b] (the arithmetic of rope_kernel) and v copied, so every row of a
// decode batch can sit at its own slot and length.
template <typename E_T>
__global__ void rope_scatter_kernel(const E_T* __restrict__ qkv, long long ldq, int H, int D, E_T* __restrict__ cache, long long ldc,
                                    int Tmax, const int* __restrict__ slot, const int* __restrict__ len, const int* __restrict__ positions,
                                    const E_T* __restrict__ cos_t, const E_T* __restrict__ sin_t) {
  using E = ElemT<E_T>;
  pdl_prologue();
  const int row = blockIdx.x;
  const int pos = positions[row];
  const int half = D >> 1;
  const int hv = half >> 3;
  const E_T* src = qkv + (long long)row * ldq;
  E_T* dst = cache + ((long long)slot[row] * Tmax + len[row]) * ldc;
  const E_T* cr = cos_t + (long long)pos * half;
  const E_T* sr = sin_t + (long long)pos * half;
  for (int idx = threadIdx.x; idx < 2 * H * hv; idx += blockDim.x) {
    const int hh = idx / hv;
    const int v = idx - hh * hv;
    const long long o = (long long)hh * D + v * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(src + o);
    const uint4 b = *reinterpret_cast<const uint4*>(src + o + half);
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(cr + v * 8));
    const uint4 s = __ldg(reinterpret_cast<const uint4*>(sr + v * 8));
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, cw[4] = {c.x, c.y, c.z, c.w}, sw[4] = {s.x, s.y, s.z, s.w};
    uint32_t oa[4], ob[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x1 = E::unpack2(aw[j]), x2 = E::unpack2(bw[j]), cs = E::unpack2(cw[j]), sn = E::unpack2(sw[j]);
      oa[j] = E::pack2(E::round(x1.x * cs.x) + E::round(-x2.x * sn.x), E::round(x1.y * cs.y) + E::round(-x2.y * sn.y));
      ob[j] = E::pack2(E::round(x2.x * cs.x) + E::round(x1.x * sn.x), E::round(x2.y * cs.y) + E::round(x1.y * sn.y));
    }
    *reinterpret_cast<uint4*>(dst + o) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(dst + o + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
  }
  const int d = H * D;
  for (int i = threadIdx.x * 8; i < d; i += blockDim.x * 8)
    *reinterpret_cast<uint4*>(dst + 2 * d + i) = *reinterpret_cast<const uint4*>(src + 2 * d + i);
}

// Paged form of rope_scatter_kernel: q is rotated in place in qkv (attention reads it there), k rotated and v copied to row
// len[b] of row b's pages (k|v rows of 2d): page page_table[slot[b]*pt_ld + (len >> page_shift)], row len & (page rows - 1).
template <typename E_T>
__global__ void rope_scatter_paged_kernel(E_T* __restrict__ qkv, long long ldq, int H, int D, E_T* __restrict__ pool, long long page_stride,
                                          long long ldc, int page_shift, const int* __restrict__ page_table, int pt_ld,
                                          const int* __restrict__ slot, const int* __restrict__ len, const int* __restrict__ positions,
                                          const E_T* __restrict__ cos_t, const E_T* __restrict__ sin_t) {
  using E = ElemT<E_T>;
  pdl_prologue();
  const int row = blockIdx.x;
  const int pos = positions[row];
  const int n = len[row];
  const int half = D >> 1;
  const int hv = half >> 3;
  const int d = H * D;
  E_T* src = qkv + (long long)row * ldq;
  E_T* dst = pool + (long long)page_table[(long long)slot[row] * pt_ld + (n >> page_shift)] * page_stride +
             (long long)(n & ((1 << page_shift) - 1)) * ldc;
  const E_T* cr = cos_t + (long long)pos * half;
  const E_T* sr = sin_t + (long long)pos * half;
  for (int idx = threadIdx.x; idx < 2 * H * hv; idx += blockDim.x) {
    const int hh = idx / hv;
    const int v = idx - hh * hv;
    const long long o = (long long)hh * D + v * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(src + o);
    const uint4 b = *reinterpret_cast<const uint4*>(src + o + half);
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(cr + v * 8));
    const uint4 s = __ldg(reinterpret_cast<const uint4*>(sr + v * 8));
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, cw[4] = {c.x, c.y, c.z, c.w}, sw[4] = {s.x, s.y, s.z, s.w};
    uint32_t oa[4], ob[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x1 = E::unpack2(aw[j]), x2 = E::unpack2(bw[j]), cs = E::unpack2(cw[j]), sn = E::unpack2(sw[j]);
      oa[j] = E::pack2(E::round(x1.x * cs.x) + E::round(-x2.x * sn.x), E::round(x1.y * cs.y) + E::round(-x2.y * sn.y));
      ob[j] = E::pack2(E::round(x2.x * cs.x) + E::round(x1.x * sn.x), E::round(x2.y * cs.y) + E::round(x1.y * sn.y));
    }
    E_T* out = hh < H ? src + o : dst + (o - d);                 // q heads in place, k heads to the page row
    *reinterpret_cast<uint4*>(out) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(out + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
  }
  for (int i = threadIdx.x * 8; i < d; i += blockDim.x * 8)
    *reinterpret_cast<uint4*>(dst + d + i) = *reinterpret_cast<const uint4*>(src + 2 * d + i);
}

// ------------------------------------------------------------------ embedding splice
// out[b, t, :] = table[ids[b, t']] for text positions; image rows are left untouched (the
// mm_projector GEMM writes them directly through its row remap).  ids layout [B, L] with
// the single IMAGE placeholder at index img_pos; output T = L - 1 + n_img rows per sample.
__global__ void embed_splice_kernel(const long long* __restrict__ ids, const bf16* __restrict__ table, bf16* __restrict__ out,
                                    int B, int L, int img_pos, int n_img, int d, int vocab) {
  const int T = L - 1 + n_img;
  const int b = blockIdx.y;
  const int j = blockIdx.x;   // index over L text slots
  if (j == img_pos) return;
  const int t = j < img_pos ? j : j - 1 + n_img;
  long long id = ids[(long long)b * L + j];
  if (id < 0 || id >= vocab) id = 0;
  const uint4* src = reinterpret_cast<const uint4*>(table + id * d);
  uint4* dst = reinterpret_cast<uint4*>(out + ((long long)b * T + t) * d);
  for (int i = threadIdx.x; i < (d >> 3); i += blockDim.x) dst[i] = __ldg(src + i);
}

// gather rows: out[i,:] = table[idx[i],:]
__global__ void gather_rows_kernel(const long long* __restrict__ idx, const bf16* __restrict__ table, long long ldt,
                                   bf16* __restrict__ out, long long ldo, int n, int d, long long nrows_table) {
  const int i = blockIdx.x;
  if (i >= n) return;
  long long r = idx[i];
  if (r < 0 || r >= nrows_table) r = 0;
  const uint4* src = reinterpret_cast<const uint4*>(table + r * ldt);
  uint4* dst = reinterpret_cast<uint4*>(out + (long long)i * ldo);
  for (int k = threadIdx.x; k < (d >> 3); k += blockDim.x) dst[k] = __ldg(src + k);
}

// ------------------------------------------------------------------ patchify (im2col for stride==kernel conv)
// pixels [B,3,S,S] (bf16) -> A [B*g*g, Kpad], k = c*P*P + py*P + px (matches conv weight.view(C_out,-1)), zero padded.
__global__ void patchify_kernel(const bf16* __restrict__ px, bf16* __restrict__ A, int B, int S, int P, int Kpad) {
  const int g = S / P;
  const long long row = blockIdx.x;            // b*g*g + gy*g + gx
  const int b = row / (g * g);
  const int r = row - (long long)b * g * g;
  const int gy = r / g, gx = r - gy * g;
  const int K = 3 * P * P;
  bf16* dst = A + row * Kpad;
  for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
    bf16 v = f2bf(0.f);
    if (k < K) {
      const int c = k / (P * P);
      const int rr = k - c * P * P;
      const int py = rr / P, pxx = rr - py * P;
      v = px[(((long long)b * 3 + c) * S + (gy * P + py)) * S + (gx * P + pxx)];
    }
    dst[k] = v;
  }
}

// x[b,0,:] = cls + pos[0]; x[b,1+i,:] = T(x[b,1+i,:]) + pos[1+i]   (T add like the reference)
template <typename T>
__global__ void vit_add_pos_kernel(T* __restrict__ x, const T* __restrict__ cls, const T* __restrict__ pos, int B,
                                   int S, int C) {
  using E = ElemT<T>;
  const long long row = blockIdx.x;   // b*S + s
  const int s = row % S;
  T* xr = x + row * C;
  const T* pr = pos + (long long)s * C;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float a = (s == 0) ? E::to_f(cls[i]) : E::to_f(xr[i]);
    xr[i] = E::from_f(a + E::to_f(pr[i]));
  }
}

// ------------------------------------------------------------------ OWL token merge
// y[b,i,:] = LN2( LN1(x[b,1+i,:]) * LN1(x[b,0,:]) )     (owlvit.py:128-138), LN1 = post_layernorm, LN2 = layer_norm
// one block per output token; C <= 1024
__global__ void __launch_bounds__(128) owl_merge_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w1,
                                                        const bf16* __restrict__ b1, const bf16* __restrict__ w2,
                                                        const bf16* __restrict__ b2, bf16* __restrict__ y, int B, int S,
                                                        int C, float eps) {
  __shared__ float red[32];
  const int n = S - 1;
  const long long o = blockIdx.x;       // b*n + i
  const int b = o / n;
  const int i = o - (long long)b * n;
  const bf16* xt = x + ((long long)b * S + 1 + i) * C;
  const bf16* xc = x + ((long long)b * S) * C;
  float t[8], c[8];
  float st = 0.f, sc = 0.f;
  int cnt = 0;
  for (int k = threadIdx.x; k < C; k += 128, ++cnt) {
    t[cnt] = bf2f(xt[k]); c[cnt] = bf2f(xc[k]);
    st += t[cnt]; sc += c[cnt];
  }
  const float mt = block_sum(st, red) / C;
  const float mc = block_sum(sc, red) / C;
  float vt = 0.f, vc = 0.f;
  for (int j = 0; j < cnt; ++j) { float d = t[j] - mt; vt += d * d; d = c[j] - mc; vc += d * d; }
  const float rt = rsqrtf(block_sum(vt, red) / C + eps);
  const float rc = rsqrtf(block_sum(vc, red) / C + eps);
  float m[8];
  float sm = 0.f;
  cnt = 0;
  for (int k = threadIdx.x; k < C; k += 128, ++cnt) {
    const float a = rbf((t[cnt] - mt) * rt * bf2f(w1[k]) + bf2f(b1[k]));
    const float cc = rbf((c[cnt] - mc) * rc * bf2f(w1[k]) + bf2f(b1[k]));
    m[cnt] = rbf(a * cc);
    sm += m[cnt];
  }
  const float mm = block_sum(sm, red) / C;
  float vm = 0.f;
  for (int j = 0; j < cnt; ++j) { float d = m[j] - mm; vm += d * d; }
  const float rm = rsqrtf(block_sum(vm, red) / C + eps);
  cnt = 0;
  bf16* yr = y + o * C;
  for (int k = threadIdx.x; k < C; k += 128, ++cnt) yr[k] = f2bf((m[cnt] - mm) * rm * bf2f(w2[k]) + bf2f(b2[k]));
}

// y[r,:] = a[r,:] + b[r % bmod, :]   (T = bf16 / f16)
template <typename T>
__global__ void add_rows_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, long long rows,
                                int cols, long long bmod) {
  using E = ElemT<T>;
  const long long n8 = (long long)rows * (cols >> 3);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (cols >> 3);
    const int c8 = i - r * (cols >> 3);
    uint4 ua = reinterpret_cast<const uint4*>(a)[i];
    uint4 ub = __ldg(reinterpret_cast<const uint4*>(b) + (r % bmod) * (cols >> 3) + c8);
    float2 p, q;
    uint4 o;
    p = E::unpack2(ua.x); q = E::unpack2(ub.x); o.x = E::pack2(p.x + q.x, p.y + q.y);
    p = E::unpack2(ua.y); q = E::unpack2(ub.y); o.y = E::pack2(p.x + q.x, p.y + q.y);
    p = E::unpack2(ua.z); q = E::unpack2(ub.z); o.z = E::pack2(p.x + q.x, p.y + q.y);
    p = E::unpack2(ua.w); q = E::unpack2(ub.w); o.w = E::pack2(p.x + q.x, p.y + q.y);
    reinterpret_cast<uint4*>(y)[i] = o;
  }
}

// fp32 -> T casts (pixel upload path)
template <typename T>
__global__ void cast_f32_kernel(const float* __restrict__ x, T* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = ElemT<T>::from_f(x[i]);
}

// (v, i) replaces (best, bi) as the running argmax.  torch.argmax's order: NaN is larger than every number (the first NaN
// wins), ties go to the smaller index.  So a row of NaN or of -inf still returns an index inside the row.
__device__ __forceinline__ bool argmax_better(float v, int i, float best, int bi) {
  const bool vn = v != v, bn = best != best;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > best || (v == best && i < bi);
}

// argmax over rows of fp32 logits [rows, n] -> idx (int32) and value (= x[idx]), with torch.argmax's semantics (above)
__global__ void __launch_bounds__(256) argmax_rows_kernel(const float* __restrict__ x, long long ld, int n, int* __restrict__ idx,
                                                          float* __restrict__ val) {
  __shared__ float sv[8];
  __shared__ int si[8];
  const float* xr = x + (long long)blockIdx.x * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v = xr[i];
    if (argmax_better(v, i, best, bi)) { best = v; bi = i; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (blockDim.x >> 5); ++w)
      if (argmax_better(sv[w], si[w], best, bi)) { best = sv[w]; bi = si[w]; }
    idx[blockIdx.x] = bi;
    if (val) val[blockIdx.x] = best;
  }
}

// negative log-likelihood of label[r] under softmax(logits[r, :]) (fp32): lse - logit[label]
//   (CrossEntropyLoss of vstar_bench_eval.py:154-159, one row per option token)
__global__ void __launch_bounds__(256) nll_rows_kernel(const float* __restrict__ x, long long ld, int n, const long long* __restrict__ labels,
                                                       float* __restrict__ out) {
  __shared__ float red[32];
  const float* xr = x + (long long)blockIdx.x * ld;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, xr[i]);
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += expf(xr[i] - mx);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const long long lb = labels[blockIdx.x];
    out[blockIdx.x] = (lb >= 0 && lb < n) ? (logf(s) + mx - xr[lb]) : 0.f;
  }
}

}  // namespace

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

template <typename T>
static int layernorm(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int rows,
                                  int cols, float eps, int act, void* stream) {
  VSB_CHECK_ARG(x && w && b && y, "vsb_layernorm_bf16: null pointer");
  VSB_CHECK_ARG(cols % 8 == 0 && cols <= 128 * 8 * 4 && ldx % 8 == 0 && ldy % 8 == 0, "vsb_layernorm_bf16: cols=%d must be a multiple of 8 and <= 4096", cols);
  if (rows <= 0) return VSB_OK;
  const int blocks = (rows + 3) / 4;
  if (cols <= 1024)
    layernorm_kernel<4, T><<<blocks, 128, 0, STREAM(stream)>>>((const T*)x, ldx, (const T*)w, (const T*)b, (T*)y, ldy, rows, cols, eps, act);
  else
    layernorm_kernel<16, T><<<blocks, 128, 0, STREAM(stream)>>>((const T*)x, ldx, (const T*)w, (const T*)b, (T*)y, ldy, rows, cols, eps, act);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename T>
static int rmsnorm(const void* x, long long ldx, const void* w, void* y, long long ldy, int rows, int cols,
                                float eps, void* stream) {
  VSB_CHECK_ARG(x && w && y, "vsb_rmsnorm_bf16: null pointer");
  VSB_CHECK_ARG(cols % 8 == 0 && cols <= 128 * 8 * 4 && ldx % 8 == 0 && ldy % 8 == 0, "vsb_rmsnorm_bf16: cols=%d must be a multiple of 8 and <= 4096", cols);
  if (rows <= 0) return VSB_OK;
  const int blocks = (rows + 3) / 4;
  if (rows <= 32 && cols >= 2048 && cols <= 8192 && !vsb_batch_invariant()) {
    VSB_CUDA(vsb_launch_pdl(rmsnorm_row_kernel<T>, dim3(rows), dim3(256), 0, STREAM(stream), 1, (const T*)x, ldx, (const T*)w, (T*)y,
                            ldy, cols, eps));
    return VSB_OK;
  }
  if (cols <= 1024)
    rmsnorm_kernel<4, T><<<blocks, 128, 0, STREAM(stream)>>>((const T*)x, ldx, (const T*)w, (T*)y, ldy, rows, cols, eps);
  else
    rmsnorm_kernel<16, T><<<blocks, 128, 0, STREAM(stream)>>>((const T*)x, ldx, (const T*)w, (T*)y, ldy, rows, cols, eps);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

// sum of squares of every row (fp32), the input side of a folded RMSNorm (vsb_gemm_rowscale_bf16 with sq_in_chunks = 1);
// one warp per row, fixed summation order
template <typename T>
__global__ void __launch_bounds__(128) rowsq_kernel(const T* __restrict__ x, long long ldx, float* __restrict__ out, int rows, int cols) {
  using E = ElemT<T>;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const T* xr = x + (long long)row * ldx;
  float s = 0.f;
  for (int c = lane * 8; c < cols; c += 256) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
    float2 t;
    t = E::unpack2(v.x); s = fmaf(t.x, t.x, s); s = fmaf(t.y, t.y, s);
    t = E::unpack2(v.y); s = fmaf(t.x, t.x, s); s = fmaf(t.y, t.y, s);
    t = E::unpack2(v.z); s = fmaf(t.x, t.x, s); s = fmaf(t.y, t.y, s);
    t = E::unpack2(v.w); s = fmaf(t.x, t.x, s); s = fmaf(t.y, t.y, s);
  }
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

template <typename T>
static int rowsq(const void* x, long long ldx, void* out_f32, int rows, int cols, void* stream) {
  VSB_CHECK_ARG(x && out_f32 && cols % 8 == 0 && ldx % 8 == 0, "vsb_rowsq_bf16: bad args (cols, ldx multiples of 8)");
  if (rows <= 0) return VSB_OK;
  rowsq_kernel<T><<<(rows + 3) / 4, 128, 0, STREAM(stream)>>>((const T*)x, ldx, (float*)out_f32, rows, cols);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename E_T>
static int rope(void* qkv, long long ld, int rows, int T, int H, int D, int pos0, const void* cos_table,
                             const void* sin_table, const void* positions, long long group_stride, long long group_offset,
                             void* stream) {
  VSB_CHECK_ARG(qkv && cos_table && sin_table && rows >= 0 && T > 0 && H > 0 && D % 16 == 0 && ld % 8 == 0, "vsb_rope_bf16: bad args (D % 16, ld % 8)");
  if (rows == 0) return VSB_OK;
  VSB_CUDA(vsb_launch_pdl(rope_kernel<E_T>, dim3(rows), dim3(256), 0, STREAM(stream), 1, (E_T*)qkv, ld, rows, T, H, D, pos0,
                          (const E_T*)cos_table, (const E_T*)sin_table, (const int*)positions, group_stride, group_offset));
  return VSB_OK;
}

template <typename E_T>
static int rope_scatter(const void* qkv, long long ldq, int B, int H, int D, void* cache, long long ldc, int Tmax, const void* slot,
                        const void* len, const void* positions, const void* cos_table, const void* sin_table, void* stream) {
  VSB_CHECK_ARG(qkv && cache && slot && len && positions && cos_table && sin_table, "vsb_rope_scatter: null pointer");
  VSB_CHECK_ARG(B >= 0 && H > 0 && Tmax > 0 && D % 16 == 0 && ldq % 8 == 0 && ldc % 8 == 0 && ldq >= 3LL * H * D && ldc >= 3LL * H * D,
                "vsb_rope_scatter: bad args (D %% 16, ld %% 8, ld >= 3*H*D)");
  if (B == 0) return VSB_OK;
  VSB_CUDA(vsb_launch_pdl(rope_scatter_kernel<E_T>, dim3(B), dim3(256), 0, STREAM(stream), 1, (const E_T*)qkv, ldq, H, D, (E_T*)cache, ldc,
                          Tmax, (const int*)slot, (const int*)len, (const int*)positions, (const E_T*)cos_table, (const E_T*)sin_table));
  return VSB_OK;
}

extern "C" int vsb_rope_scatter(const void* qkv, long long ldq, int B, int H, int D, void* cache, long long ldc, int Tmax, const void* slot_i32,
                                const void* len_i32, const void* pos_i32, const void* cos_table, const void* sin_table, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_rope_scatter: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  return dtype == VSB_DTYPE_F16 ? rope_scatter<half>(qkv, ldq, B, H, D, cache, ldc, Tmax, slot_i32, len_i32, pos_i32, cos_table, sin_table, stream)
                                : rope_scatter<bf16>(qkv, ldq, B, H, D, cache, ldc, Tmax, slot_i32, len_i32, pos_i32, cos_table, sin_table, stream);
}

template <typename E_T>
static int rope_scatter_paged(void* qkv, long long ldq, int B, int H, int D, void* pool, long long page_stride, long long ldc, int page_rows,
                              const void* page_table, int pt_ld, const void* slot, const void* len, const void* positions,
                              const void* cos_table, const void* sin_table, void* stream) {
  VSB_CHECK_ARG(qkv && pool && page_table && slot && len && positions && cos_table && sin_table, "vsb_rope_scatter_paged: null pointer");
  VSB_CHECK_ARG(B >= 0 && H > 0 && pt_ld > 0 && D % 16 == 0 && ldq % 8 == 0 && ldc % 8 == 0 && page_stride % 8 == 0 && ldq >= 3LL * H * D &&
                    ldc >= 2LL * H * D && page_stride >= (long long)page_rows * ldc,
                "vsb_rope_scatter_paged: bad args (D %% 16, ld %% 8, ldq >= 3*H*D, ldc >= 2*H*D, page_stride >= page_rows*ldc)");
  VSB_CHECK_ARG(page_rows >= 16 && (page_rows & (page_rows - 1)) == 0, "vsb_rope_scatter_paged: page_rows %d is not a power of two >= 16",
                page_rows);
  if (B == 0) return VSB_OK;
  VSB_CUDA(vsb_launch_pdl(rope_scatter_paged_kernel<E_T>, dim3(B), dim3(256), 0, STREAM(stream), 1, (E_T*)qkv, ldq, H, D, (E_T*)pool, page_stride,
                          ldc, __builtin_ctz((unsigned)page_rows), (const int*)page_table, pt_ld, (const int*)slot, (const int*)len,
                          (const int*)positions, (const E_T*)cos_table, (const E_T*)sin_table));
  return VSB_OK;
}

extern "C" int vsb_rope_scatter_paged(void* qkv, long long ldq, int B, int H, int D, void* pool, long long page_stride, long long ldc,
                                      int page_rows, const void* page_table_i32, int pt_ld, const void* slot_i32, const void* len_i32,
                                      const void* pos_i32, const void* cos_table, const void* sin_table, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_rope_scatter_paged: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  return dtype == VSB_DTYPE_F16
             ? rope_scatter_paged<half>(qkv, ldq, B, H, D, pool, page_stride, ldc, page_rows, page_table_i32, pt_ld, slot_i32, len_i32, pos_i32,
                                        cos_table, sin_table, stream)
             : rope_scatter_paged<bf16>(qkv, ldq, B, H, D, pool, page_stride, ldc, page_rows, page_table_i32, pt_ld, slot_i32, len_i32, pos_i32,
                                        cos_table, sin_table, stream);
}

extern "C" int vsb_embed_splice_bf16(const void* ids, const void* table, void* out, int B, int L, int img_pos, int n_img, int d,
                                     int vocab, void* stream) {
  VSB_CHECK_ARG(ids && table && out && d % 8 == 0 && img_pos >= 0 && img_pos < L, "vsb_embed_splice_bf16: bad args");
  dim3 grid(L, B);
  embed_splice_kernel<<<grid, 128, 0, STREAM(stream)>>>((const long long*)ids, (const bf16*)table, (bf16*)out, B, L, img_pos, n_img, d, vocab);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_gather_rows_bf16(const void* idx, const void* table, long long ldt, void* out, long long ldo, int n, int d,
                                    long long nrows_table, void* stream) {
  VSB_CHECK_ARG(idx && table && out && d % 8 == 0 && ldt % 8 == 0 && ldo % 8 == 0, "vsb_gather_rows_bf16: bad args");
  if (n <= 0) return VSB_OK;
  gather_rows_kernel<<<n, 128, 0, STREAM(stream)>>>((const long long*)idx, (const bf16*)table, ldt, (bf16*)out, ldo, n, d, nrows_table);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_patchify_bf16(const void* pixels, void* A, int B, int S, int P, int Kpad, void* stream) {
  VSB_CHECK_ARG(pixels && A && S % P == 0 && Kpad >= 3 * P * P && Kpad % 8 == 0, "vsb_patchify_bf16: bad args");
  const int g = S / P;
  patchify_kernel<<<B * g * g, 128, 0, STREAM(stream)>>>((const bf16*)pixels, (bf16*)A, B, S, P, Kpad);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename T>
static int vit_add_pos(void* x, const void* cls, const void* pos, int B, int S, int C, void* stream) {
  VSB_CHECK_ARG(x && cls && pos, "vsb_vit_add_pos_bf16: null pointer");
  vit_add_pos_kernel<T><<<B * S, 128, 0, STREAM(stream)>>>((T*)x, (const T*)cls, (const T*)pos, B, S, C);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_owl_merge_bf16(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, void* y, int B,
                                  int S, int C, float eps, void* stream) {
  VSB_CHECK_ARG(x && w1 && b1 && w2 && b2 && y && C <= 1024, "vsb_owl_merge_bf16: bad args (C<=1024)");
  owl_merge_kernel<<<B * (S - 1), 128, 0, STREAM(stream)>>>((const bf16*)x, (const bf16*)w1, (const bf16*)b1, (const bf16*)w2,
                                                            (const bf16*)b2, (bf16*)y, B, S, C, eps);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename T>
static int add_rows(const void* a, const void* b, void* y, long long rows, int cols, long long bmod, void* stream) {
  VSB_CHECK_ARG(a && b && y && cols % 8 == 0 && bmod > 0, "vsb_add_rows_bf16: bad args");
  if (rows <= 0) return VSB_OK;
  long long n8 = rows * (cols >> 3);
  int blocks = (int)((n8 + 255) / 256);
  if (blocks > vsb_num_sms() * 16) blocks = vsb_num_sms() * 16;
  add_rows_kernel<T><<<blocks, 256, 0, STREAM(stream)>>>((const T*)a, (const T*)b, (T*)y, rows, cols, bmod);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

template <typename T>
static int cast_f32(const void* x, void* y, long long n, void* stream) {
  VSB_CHECK_ARG(x && y, "vsb_cast_f32_bf16: null pointer");
  if (n <= 0) return VSB_OK;
  int blocks = (int)((n + 255) / 256);
  if (blocks > vsb_num_sms() * 16) blocks = vsb_num_sms() * 16;
  cast_f32_kernel<T><<<blocks, 256, 0, STREAM(stream)>>>((const float*)x, (T*)y, n);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_nll_rows_f32(const void* x, long long ld, int rows, int n, const void* labels_i64, void* out, void* stream) {
  VSB_CHECK_ARG(x && labels_i64 && out && n > 0, "vsb_nll_rows_f32: bad args");
  if (rows <= 0) return VSB_OK;
  nll_rows_kernel<<<rows, 256, 0, STREAM(stream)>>>((const float*)x, ld, n, (const long long*)labels_i64, (float*)out);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_argmax_rows_f32(const void* x, long long ld, int rows, int n, void* idx, void* val, void* stream) {
  VSB_CHECK_ARG(x && idx && n > 0, "vsb_argmax_rows_f32: bad args");
  if (rows <= 0) return VSB_OK;
  argmax_rows_kernel<<<rows, 256, 0, STREAM(stream)>>>((const float*)x, ld, n, (int*)idx, (float*)val);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

// ------------------------------------------------------------------ C entry points: bf16 and f16 (the VQA engine in fp16)
extern "C" int vsb_layernorm_bf16(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int rows, int cols,
                                  float eps, int act, void* stream) {
  return layernorm<bf16>(x, ldx, w, b, y, ldy, rows, cols, eps, act, stream);
}
extern "C" int vsb_layernorm_f16(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int rows, int cols,
                                 float eps, int act, void* stream) {
  return layernorm<half>(x, ldx, w, b, y, ldy, rows, cols, eps, act, stream);
}
extern "C" int vsb_rmsnorm_bf16(const void* x, long long ldx, const void* w, void* y, long long ldy, int rows, int cols, float eps, void* stream) {
  return rmsnorm<bf16>(x, ldx, w, y, ldy, rows, cols, eps, stream);
}
extern "C" int vsb_rmsnorm_f16(const void* x, long long ldx, const void* w, void* y, long long ldy, int rows, int cols, float eps, void* stream) {
  return rmsnorm<half>(x, ldx, w, y, ldy, rows, cols, eps, stream);
}
extern "C" int vsb_rowsq_bf16(const void* x, long long ldx, void* out_f32, int rows, int cols, void* stream) {
  return rowsq<bf16>(x, ldx, out_f32, rows, cols, stream);
}
extern "C" int vsb_rowsq_f16(const void* x, long long ldx, void* out_f32, int rows, int cols, void* stream) {
  return rowsq<half>(x, ldx, out_f32, rows, cols, stream);
}
extern "C" int vsb_rope_bf16(void* qkv, long long ld, int rows, int T, int H, int D, int pos0, const void* cos_table, const void* sin_table,
                             const void* positions, long long group_stride, long long group_offset, void* stream) {
  return rope<bf16>(qkv, ld, rows, T, H, D, pos0, cos_table, sin_table, positions, group_stride, group_offset, stream);
}
extern "C" int vsb_rope_f16(void* qkv, long long ld, int rows, int T, int H, int D, int pos0, const void* cos_table, const void* sin_table,
                            const void* positions, long long group_stride, long long group_offset, void* stream) {
  return rope<half>(qkv, ld, rows, T, H, D, pos0, cos_table, sin_table, positions, group_stride, group_offset, stream);
}
extern "C" int vsb_vit_add_pos_bf16(void* x, const void* cls, const void* pos, int B, int S, int C, void* stream) {
  return vit_add_pos<bf16>(x, cls, pos, B, S, C, stream);
}
extern "C" int vsb_vit_add_pos_f16(void* x, const void* cls, const void* pos, int B, int S, int C, void* stream) {
  return vit_add_pos<half>(x, cls, pos, B, S, C, stream);
}
extern "C" int vsb_add_rows_bf16(const void* a, const void* b, void* y, long long rows, int cols, long long bmod, void* stream) {
  return add_rows<bf16>(a, b, y, rows, cols, bmod, stream);
}
extern "C" int vsb_add_rows_f16(const void* a, const void* b, void* y, long long rows, int cols, long long bmod, void* stream) {
  return add_rows<half>(a, b, y, rows, cols, bmod, stream);
}
extern "C" int vsb_cast_f32_bf16(const void* x, void* y, long long n, void* stream) { return cast_f32<bf16>(x, y, n, stream); }
extern "C" int vsb_cast_f32_f16(const void* x, void* y, long long n, void* stream) { return cast_f32<half>(x, y, n, stream); }
