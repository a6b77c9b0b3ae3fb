// Post-backbone kernels of the VSM hot path: OWL-ViT class/box head epilogues, SAM mask-decoder
// upscaling helpers (bilinear x2, 3x3 im2col, hyper-network dot), the full-resolution target-cue
// heatmap (bilinear + clamp) with its reductions, and the quad-tree rectangle sums used by the search
// controller.  All HBM/L2-bound streaming kernels (coalesced, vectorised where rows are contiguous).
#include "common.cuh"
#include "vstar_b200.h"

namespace {

// ---------------------------------------------------------------- OWL class head epilogue
// y [R, ldy] fp32 = [dense0(x) (Q cols) | logit_shift | logit_scale]  (one GEMM with stacked weights)
// logit = (<y/(|y|+1e-6), q/(|q|+1e-6)> + shift) * (elu(scale) + 1)
//   (transformers/models/owlvit/modeling_owlvit.py:1043-1062); one warp per row.
__global__ void __launch_bounds__(128) owl_class_post_kernel(const float* __restrict__ y, long long ldy,
                                                             const bf16* __restrict__ query, long long ldq, int rows_per_crop,
                                                             long long R, int Q, int quant_bf16, float* __restrict__ logits,
                                                             float* __restrict__ scores) {
  const long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= R) return;
  const int b = row / rows_per_crop;
  const float* yr = y + row * ldy;
  const bf16* qr = query + (long long)b * ldq;
  float yy = 0.f, qq = 0.f, yq = 0.f;
  for (int i = lane; i < Q; i += 32) {
    const float a = yr[i], c = bf2f(qr[i]);
    yy += a * a; qq += c * c; yq += a * c;
  }
  yy = warp_sum(yy); qq = warp_sum(qq); yq = warp_sum(yq);
  if (lane == 0) {
    const float dot = yq / ((sqrtf(yy) + 1e-6f) * (sqrtf(qq) + 1e-6f));
    const float shift = yr[Q], sc = yr[Q + 1];
    const float scale = (sc > 0.f ? sc : expm1f(sc)) + 1.f;
    float l = (dot + shift) * scale;
    // quant_bf16: the reference model runs in bf16, so pred_logits and .sigmoid() are bf16 VALUES (visual_search.py:145,
    // :223-224): thresholds, argmax ties (first index wins) and all_valid_boxes are decided on the rounded numbers
    if (quant_bf16) l = rbf(l);
    logits[row] = l;
    if (scores) {
      const float sg = 1.f / (1.f + expf(-l));
      scores[row] = quant_bf16 ? rbf(sg) : sg;
    }
  }
}

// boxes = sigmoid(y[:, :4] + box_bias[row % rows_per_crop])   (owlvit.py:79-100)
__global__ void owl_box_post_kernel(const float* __restrict__ y, long long ldy, const float* __restrict__ bias, int rows_per_crop,
                                    long long R, int quant_bf16, float* __restrict__ boxes) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= R * 4) return;
  const long long row = i >> 2;
  const int c = i & 3;
  float v = y[row * ldy + c];
  const float b = bias[(row % rows_per_crop) * 4 + c];
  if (quant_bf16) {       // bf16 head output, in-place `+= box_bias` (stays bf16), bf16 sigmoid (owlvit.py:95-99)
    v = rbf(rbf(v) + b);
    boxes[i] = rbf(1.f / (1.f + expf(-v)));
  } else {
    boxes[i] = 1.f / (1.f + expf(-(v + b)));
  }
}

// ---------------------------------------------------------------- bilinear x2, NHWC bf16 (fp32 math, bf16 out)
// torch.nn.functional.interpolate(x.float(), scale_factor=2, mode="bilinear").to(bf16)
//   (/root/reference/VisualSearch/model/segment_anything/modeling/mask_decoder.py:24-27)
__global__ void upsample2x_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int H, int W, int C) {
  const int OH = 2 * H, OW = 2 * W;
  const long long pix = blockIdx.x;             // b*OH*OW + oy*OW + ox
  const int ox = pix % OW;
  const int oy = (pix / OW) % OH;
  const int b = pix / ((long long)OW * OH);
  float sy = 0.5f * (oy + 0.5f) - 0.5f; if (sy < 0.f) sy = 0.f;
  float sx = 0.5f * (ox + 0.5f) - 0.5f; if (sx < 0.f) sx = 0.f;
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const bf16* p00 = x + (((long long)b * H + y0) * W + x0) * C;
  const bf16* p01 = x + (((long long)b * H + y0) * W + x1) * C;
  const bf16* p10 = x + (((long long)b * H + y1) * W + x0) * C;
  const bf16* p11 = x + (((long long)b * H + y1) * W + x1) * C;
  bf16* o = y + pix * C;
  for (int c = threadIdx.x * 2; c < C; c += blockDim.x * 2) {
    const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p00 + c));
    const float2 bb = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p01 + c));
    const float2 cc = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p10 + c));
    const float2 d = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p11 + c));
    const float r0 = hy * (hx * a.x + lx * bb.x) + ly * (hx * cc.x + lx * d.x);
    const float r1 = hy * (hx * a.y + lx * bb.y) + ly * (hx * cc.y + lx * d.y);
    *reinterpret_cast<uint32_t*>(o + c) = pack_bf16x2(r0, r1);
  }
}

// ---------------------------------------------------------------- im2col for 3x3 / pad 1 / stride 1, NHWC bf16
// A[(b,y,x), (ky*3+kx)*C + c] = X[b, y+ky-1, x+kx-1, c] (0 outside); conv weight must be permuted to [Cout, ky, kx, Cin].
__global__ void im2col3x3_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ A, int B, int H, int W, int C) {
  const long long pix = blockIdx.x;
  const int ox = pix % W;
  const int oy = (pix / W) % H;
  const int b = pix / ((long long)W * H);
  const int c8 = C >> 3;
  uint4* dst = reinterpret_cast<uint4*>(A + pix * 9 * C);
  for (int i = threadIdx.x; i < 9 * c8; i += blockDim.x) {
    const int tap = i / c8, cc = i - tap * c8;
    const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = *(reinterpret_cast<const uint4*>(x + (((long long)b * H + iy) * W + ix) * C) + cc);
    dst[i] = v;
  }
}

// ---------------------------------------------------------------- masks[b,p] = sum_c hyper[b,c] * up[b,p,c]
//   (mask_decoder.py:178-181, mask token 0 only since multimask_output=False)
__global__ void mask_dot_kernel(const bf16* __restrict__ up, const bf16* __restrict__ hyper, float* __restrict__ out, int B,
                                long long P, int C) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * P) return;
  const int b = i / P;
  const bf16* u = up + i * C;
  const bf16* hrow = hyper + (long long)b * C;
  float s = 0.f;
  for (int c = 0; c < C; c += 8) {
    uint4 a = *reinterpret_cast<const uint4*>(u + c);
    uint4 hh = __ldg(reinterpret_cast<const uint4*>(hrow + c));
    float2 p, q;
    p = unpack_bf16x2(a.x); q = unpack_bf16x2(hh.x); s += p.x * q.x + p.y * q.y;
    p = unpack_bf16x2(a.y); q = unpack_bf16x2(hh.y); s += p.x * q.x + p.y * q.y;
    p = unpack_bf16x2(a.z); q = unpack_bf16x2(hh.z); s += p.x * q.x + p.y * q.y;
    p = unpack_bf16x2(a.w); q = unpack_bf16x2(hh.w); s += p.x * q.x + p.y * q.y;
  }
  out[i] = s;
}

// ---------------------------------------------------------------- target-cue heatmap
// F.interpolate(low_res.float(), (h, w), mode="bilinear", align_corners=False) then clamp(min=0)
//   (/root/reference/VisualSearch/model/VSM.py:534-537; /root/reference/visual_search.py:223-224)
// Same arithmetic order as ATen's upsample_bilinear2d (fp32 accscalar).  Also emits per-block partial
// (max, min, sum) so the search controller never has to re-read the H x W map for its statistics.
// One pixel of F.interpolate(low, (h, w), mode="bilinear", align_corners=False) (+ clamp), same expression as ATen's
// upsample_bilinear2d (fp32 accscalar; nvcc contracts it into FMAs as it does for ATen).  Deliberately NOT inlined: every
// kernel that evaluates the map (materialising heatmap_kernel, the fused statistics / rectangle-sum kernels of the crop
// records) calls this one compiled body, so they all produce bit-identical values.
struct HeatGeom {
  const float* low;
  int LH, LW;
  float rh, rw;
  int do_clamp;
};
__device__ __noinline__ float heat_px(const float* __restrict__ low, int LH, int LW, float rh, float rw, int do_clamp, int oy, int ox) {
  float sy = rh * (oy + 0.5f) - 0.5f; if (sy < 0.f) sy = 0.f;
  float sx = rw * (ox + 0.5f) - 0.5f; if (sx < 0.f) sx = 0.f;
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < LH - 1 ? 1 : 0), x1 = x0 + (x0 < LW - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0, hy = 1.f - ly, hx = 1.f - lx;
  float v = hy * (hx * low[y0 * LW + x0] + lx * low[y0 * LW + x1]) + ly * (hx * low[y1 * LW + x0] + lx * low[y1 * LW + x1]);
  if (do_clamp) v = fmaxf(v, 0.f);
  return v;
}
__device__ __forceinline__ float heat_px(const HeatGeom& g, int oy, int ox) { return heat_px(g.low, g.LH, g.LW, g.rh, g.rw, g.do_clamp, oy, ox); }

__global__ void __launch_bounds__(256) heatmap_kernel(const float* __restrict__ low, int LH, int LW, float* __restrict__ out, int h,
                                                      int w, int do_clamp, float* __restrict__ partial) {
  __shared__ float smax[8], smin[8], ssum[8];
  HeatGeom g{low, LH, LW, (float)LH / (float)h, (float)LW / (float)w, do_clamp};
  const long long n = (long long)h * w;
  float mx = -INFINITY, mn = INFINITY, sm = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int oy = i / w, ox = i - (long long)oy * w;
    const float v = heat_px(g, oy, ox);
    out[i] = v;
    mx = fmaxf(mx, v); mn = fminf(mn, v); sm += v;
  }
  mx = warp_max(mx); mn = warp_min(mn); sm = warp_sum(sm);
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { smax[wid] = mx; smin[wid] = mn; ssum[wid] = sm; }
  __syncthreads();
  if (threadIdx.x == 0 && partial) {
    for (int k = 1; k < 8; ++k) { mx = fmaxf(mx, smax[k]); mn = fminf(mn, smin[k]); sm += ssum[k]; }
    partial[blockIdx.x * 3 + 0] = mx; partial[blockIdx.x * 3 + 1] = mn; partial[blockIdx.x * 3 + 2] = sm;
  }
}

__global__ void __launch_bounds__(256) stats_final_kernel(const float* __restrict__ partial, int n, float* __restrict__ out3) {
  __shared__ float smax[8], smin[8];
  __shared__ double ssum[8];
  float mx = -INFINITY, mn = INFINITY;
  double sm = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    mx = fmaxf(mx, partial[i * 3]); mn = fminf(mn, partial[i * 3 + 1]); sm += (double)partial[i * 3 + 2];
  }
  mx = warp_max(mx); mn = warp_min(mn);
  for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { smax[wid] = mx; smin[wid] = mn; ssum[wid] = sm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) { mx = fmaxf(mx, smax[k]); mn = fminf(mn, smin[k]); sm += ssum[k]; }
    out3[0] = mx; out3[1] = mn; out3[2] = (float)sm;
  }
}

// ---------------------------------------------------------------- rectangle sums of the normalised heatmap
// out[r] = sum over rect r of  (hm[y,x] - min) / (max - min)     (normalize_score folded in; 0 for a flat map)
//   (/root/reference/visual_search.py:255-275).  grid = (RECT_CHUNKS, nrects): every block reduces a band of rows of its
// rectangle (coalesced row segments, fp32 per-thread partials flushed to fp64 every 64 elements), then a tiny second kernel
// combines the RECT_CHUNKS partials per rectangle in a fixed order (deterministic).
constexpr int RECT_CHUNKS = 64;
// normalize_score per element, IEEE ops like torch: (v - min) / (max - min); 0 for a flat map (visual_search.py:268-275)
__device__ __forceinline__ float norm_px(float v, float mn, float den) {
  return den != 0.f ? __fdiv_rn(__fadd_rn(v, -mn), den) : 0.f;
}

__global__ void __launch_bounds__(256) rect_sums_partial_kernel(const float* __restrict__ hm, int h, int w, const int* __restrict__ rects,
                                                                const float* __restrict__ stats, double* __restrict__ partial) {
  __shared__ double red[8];
  const int r = blockIdx.y, chunk = blockIdx.x;
  int x0 = rects[r * 4 + 0], y0 = rects[r * 4 + 1], rw = rects[r * 4 + 2], rh = rects[r * 4 + 3];
  int x1 = x0 + rw, y1 = y0 + rh;
  if (x0 < 0) x0 = 0; if (y0 < 0) y0 = 0; if (x1 > w) x1 = w; if (y1 > h) y1 = h;
  const float mx = stats[0], mn = stats[1];
  const float den = (mx != mn) ? __fadd_rn(mx, -mn) : 0.f;     // 0 = flat map: normalize_score returns all zeros
  const float sub = mn;
  double dacc = 0.0;
  if (x1 > x0 && y1 > y0) {
    const int rows = y1 - y0;
    const int per = (rows + RECT_CHUNKS - 1) / RECT_CHUNKS;
    const int ya = y0 + chunk * per;
    const int yb = min(y1, ya + per);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int yy = ya + warp; yy < yb; yy += 8) {           // one warp per row: coalesced
      const float* row = hm + (long long)yy * w;
      float acc = 0.f;
      int k = 0;
      for (int xx = x0 + lane; xx < x1; xx += 32) {
        acc = __fadd_rn(acc, norm_px(row[xx], sub, den));
        if (++k == 64) { dacc += acc; acc = 0.f; k = 0; }
      }
      dacc += acc;
    }
  }
  for (int o = 16; o > 0; o >>= 1) dacc += __shfl_xor_sync(0xffffffffu, dacc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < 8; ++q) dacc += red[q];
    partial[(long long)r * RECT_CHUNKS + chunk] = dacc;
  }
}

__global__ void rect_sums_final_kernel(const double* __restrict__ partial, int nrects, double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nrects) return;
  double s = 0.0;
  for (int c = 0; c < RECT_CHUNKS; ++c) s += partial[(long long)r * RECT_CHUNKS + c];
  out[r] = s;
}

// ---------------------------------------------------------------- crop records (SURVEY.md section 8e)
// Everything the search controller consumes from ONE crop evaluation, as a fixed-size fp32 record produced on the device:
//   [0] best sigmoid score  [1..4] its box (cxcywh)  [5] #rows P  [6] #rows with score > 0.5  [7] best row index (-1: no
//   finite score)  [8..10] (max, min, sum) of the clamped full-resolution target-cue map  [11] #rectangle sums
//   [12..75] the first 16 boxes with score > 0.5 in row order  [76..] sums of the min-max-normalised map over the crop and
//   every descendant sub-patch of the quad-tree below it (the ancestor-chain terms of visual_search.py:453-462).
// The H x W map itself is never written: statistics and rectangle sums are evaluated straight from the 192 x 192 low-res mask
// with the same per-pixel arithmetic as heatmap_kernel / rect_sums_partial_kernel (bit-identical results).
constexpr int REC_TOP = 0, REC_BOX = 1, REC_NROWS = 5, REC_NVALID = 6, REC_TOPIDX = 7, REC_MAX = 8, REC_MIN = 9, REC_SUM = 10,
              REC_NRECT = 11, REC_VALID = 12, REC_MAXVALID = 16, REC_PYR = 76;
constexpr int STAT_CHUNKS = 64;

// one block per crop: argmax (first index wins ties, like torch.argmax), count and compact the rows above 0.5
__global__ void __launch_bounds__(256) pack_detections_kernel(const float* __restrict__ scores, const float* __restrict__ boxes, int P,
                                                              float* __restrict__ rec, long long R) {
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ int scount[8];
  const int c = blockIdx.x;
  const float* sc = scores + (long long)c * P;
  const float4* bx = reinterpret_cast<const float4*>(boxes) + (long long)c * P;
  float* out = rec + (long long)c * R;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const float v = sc[i];
    if (v > best) { best = v; bi = i; }           // strided scan keeps the smallest index per thread for equal values
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { sv[wid] = best; si[wid] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k)
      if (sv[k] > best || (sv[k] == best && si[k] < bi)) { best = sv[k]; bi = si[k]; }
    const bool ok = bi != 0x7fffffff;
    out[REC_TOP] = ok ? best : nanf("");
    const float4 b = ok ? bx[bi] : make_float4(0.f, 0.f, 0.f, 0.f);
    out[REC_BOX + 0] = b.x; out[REC_BOX + 1] = b.y; out[REC_BOX + 2] = b.z; out[REC_BOX + 3] = b.w;
    out[REC_NROWS] = (float)P;
    out[REC_TOPIDX] = ok ? (float)bi : -1.f;
  }
  // valid rows in index order: block-wide ordered compaction, 256 rows per pass
  int base = 0;
  for (int i0 = 0; i0 < P; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const bool v = i < P && sc[i] > 0.5f;
    const unsigned m = __ballot_sync(0xffffffffu, v);
    if (lane == 0) scount[wid] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int k = 0; k < 8; ++k) { if (k < wid) before += scount[k]; total += scount[k]; }
    const int slot = base + before + __popc(m & ((1u << lane) - 1u));
    if (v && slot < REC_MAXVALID) {
      const float4 b = bx[i];
      float* d = out + REC_VALID + slot * 4;
      d[0] = b.x; d[1] = b.y; d[2] = b.z; d[3] = b.w;
    }
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) out[REC_NVALID] = (float)base;
}

// job table (int32 x 8 per job): {low_ptr lo, low_ptr hi, h, w, first rect, n_rects, record row, unused}
struct HeatJob {
  const float* low;
  int h, w, rect0, nrects, row;
};
__device__ __forceinline__ HeatJob load_job(const int* __restrict__ jobs, int j) {
  const int* q = jobs + j * 8;
  HeatJob r;
  const unsigned long long p = (unsigned long long)(unsigned)q[0] | ((unsigned long long)(unsigned)q[1] << 32);
  r.low = reinterpret_cast<const float*>(p);
  r.h = q[2]; r.w = q[3]; r.rect0 = q[4]; r.nrects = q[5]; r.row = q[6];
  return r;
}

// grid (STAT_CHUNKS, n_jobs): (max, min, sum) of the clamped map over a band of rows
__global__ void __launch_bounds__(256) heat_stats_kernel(const int* __restrict__ jobs, int LH, int LW, float* __restrict__ partial) {
  __shared__ float smax[8], smin[8], ssum[8];
  const HeatJob jb = load_job(jobs, blockIdx.y);
  HeatGeom g{jb.low, LH, LW, (float)LH / (float)jb.h, (float)LW / (float)jb.w, 1};
  const int per = (jb.h + STAT_CHUNKS - 1) / STAT_CHUNKS;
  const int ya = blockIdx.x * per, yb = min(jb.h, ya + per);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float mx = -INFINITY, mn = INFINITY, sm = 0.f;
  for (int oy = ya + warp; oy < yb; oy += 8) {
    for (int ox = lane; ox < jb.w; ox += 32) {
      const float v = heat_px(g, oy, ox);
      mx = fmaxf(mx, v); mn = fminf(mn, v); sm += v;
    }
  }
  mx = warp_max(mx); mn = warp_min(mn); sm = warp_sum(sm);
  if (lane == 0) { smax[warp] = mx; smin[warp] = mn; ssum[warp] = sm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) { mx = fmaxf(mx, smax[k]); mn = fminf(mn, smin[k]); sm += ssum[k]; }
    float* o = partial + ((long long)blockIdx.y * STAT_CHUNKS + blockIdx.x) * 3;
    o[0] = mx; o[1] = mn; o[2] = sm;
  }
}

// one warp per job: combine the band partials in a fixed order and publish them in the record
__global__ void heat_stats_final_kernel(const int* __restrict__ jobs, int n_jobs, const float* __restrict__ partial, float* __restrict__ rec,
                                        long long R) {
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= n_jobs) return;
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY, mn = INFINITY;
  double sm = 0.0;
  for (int c = lane; c < STAT_CHUNKS; c += 32) {
    const float* o = partial + ((long long)j * STAT_CHUNKS + c) * 3;
    mx = fmaxf(mx, o[0]); mn = fminf(mn, o[1]); sm += (double)o[2];
  }
  mx = warp_max(mx); mn = warp_min(mn);
  for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
  if (lane == 0) {
    const HeatJob jb = load_job(jobs, j);
    float* out = rec + (long long)jb.row * R;
    out[REC_MAX] = mx; out[REC_MIN] = mn; out[REC_SUM] = (float)sm; out[REC_NRECT] = (float)jb.nrects;
  }
}

// grid (total rects, RECT_CHUNKS): band of rows of one rectangle of the normalised map, evaluated from the low-res mask.
// Same traversal / flush order as rect_sums_partial_kernel => identical sums.
__global__ void __launch_bounds__(256) heat_rects_kernel(const int* __restrict__ jobs, const int* __restrict__ rects,
                                                         const int* __restrict__ rect_job, int LH, int LW, const float* __restrict__ rec,
                                                         long long R, double* __restrict__ partial) {
  __shared__ double red[8];
  const int r = blockIdx.x, chunk = blockIdx.y;
  const HeatJob jb = load_job(jobs, rect_job[r]);
  HeatGeom g{jb.low, LH, LW, (float)LH / (float)jb.h, (float)LW / (float)jb.w, 1};
  int x0 = rects[r * 4 + 0], y0 = rects[r * 4 + 1], rw = rects[r * 4 + 2], rh = rects[r * 4 + 3];
  int x1 = x0 + rw, y1 = y0 + rh;
  if (x0 < 0) x0 = 0; if (y0 < 0) y0 = 0; if (x1 > jb.w) x1 = jb.w; if (y1 > jb.h) y1 = jb.h;
  const float* st = rec + (long long)jb.row * R;
  const float mx = st[REC_MAX], mn = st[REC_MIN];
  const float den = (mx != mn) ? __fadd_rn(mx, -mn) : 0.f;
  const float sub = mn;
  double dacc = 0.0;
  if (x1 > x0 && y1 > y0) {
    const int rows = y1 - y0;
    const int per = (rows + RECT_CHUNKS - 1) / RECT_CHUNKS;
    const int ya = y0 + chunk * per;
    const int yb = min(y1, ya + per);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int yy = ya + warp; yy < yb; yy += 8) {
      float acc = 0.f;
      int k = 0;
      for (int xx = x0 + lane; xx < x1; xx += 32) {
        acc = __fadd_rn(acc, norm_px(heat_px(g, yy, xx), sub, den));
        if (++k == 64) { dacc += acc; acc = 0.f; k = 0; }
      }
      dacc += acc;
    }
  }
  for (int o = 16; o > 0; o >>= 1) dacc += __shfl_xor_sync(0xffffffffu, dacc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < 8; ++q) dacc += red[q];
    partial[(long long)r * RECT_CHUNKS + chunk] = dacc;
  }
}

__global__ void heat_rects_final_kernel(const int* __restrict__ jobs, const int* __restrict__ rect_job, int total,
                                        const double* __restrict__ partial, float* __restrict__ rec, long long R) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total) return;
  const HeatJob jb = load_job(jobs, rect_job[r]);
  double s = 0.0;
  for (int c = 0; c < RECT_CHUNKS; ++c) s += partial[(long long)r * RECT_CHUNKS + c];
  rec[(long long)jb.row * R + REC_PYR + (r - jb.rect0)] = (float)s;      // np.float32(sum), as the controller would cast it
}

// strided 2-D copy of 16-byte vectors: dst[r, :] = src[r, :]
__global__ void copy2d_kernel(const uint4* __restrict__ src, long long lds16, uint4* __restrict__ dst, long long ldd16, long long rows,
                              int cols16) {
  const long long n = rows * cols16;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols16;
    const int c = i - r * cols16;
    dst[r * ldd16 + c] = src[r * lds16 + c];
  }
}

}  // namespace

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int vsb_owl_class_post(const void* y, long long ldy, const void* query, long long ldq, int rows_per_crop, long long R, int Q,
                                  int quant_bf16, void* logits, void* scores, void* stream) {
  VSB_CHECK_ARG(y && query && logits && Q > 0 && rows_per_crop > 0, "vsb_owl_class_post: bad args");
  if (R <= 0) return VSB_OK;
  const int blocks = (int)((R + 3) / 4);
  owl_class_post_kernel<<<blocks, 128, 0, STREAM(stream)>>>((const float*)y, ldy, (const bf16*)query, ldq, rows_per_crop, R, Q,
                                                            quant_bf16, (float*)logits, (float*)scores);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_owl_box_post(const void* y, long long ldy, const void* box_bias, int rows_per_crop, long long R, int quant_bf16,
                                void* boxes, void* stream) {
  VSB_CHECK_ARG(y && box_bias && boxes && rows_per_crop > 0, "vsb_owl_box_post: bad args");
  if (R <= 0) return VSB_OK;
  const int blocks = (int)((R * 4 + 255) / 256);
  owl_box_post_kernel<<<blocks, 256, 0, STREAM(stream)>>>((const float*)y, ldy, (const float*)box_bias, rows_per_crop, R, quant_bf16, (float*)boxes);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_upsample2x_nhwc_bf16(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  VSB_CHECK_ARG(x && y && C % 2 == 0, "vsb_upsample2x_nhwc_bf16: bad args");
  const long long pix = (long long)B * 4 * H * W;
  if (pix <= 0) return VSB_OK;
  const int threads = C / 2 < 128 ? (C / 2 < 32 ? 32 : C / 2) : 128;
  upsample2x_nhwc_kernel<<<(unsigned)pix, threads, 0, STREAM(stream)>>>((const bf16*)x, (bf16*)y, B, H, W, C);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_im2col3x3_nhwc_bf16(const void* x, void* A, int B, int H, int W, int C, void* stream) {
  VSB_CHECK_ARG(x && A && C % 8 == 0, "vsb_im2col3x3_nhwc_bf16: bad args");
  const long long pix = (long long)B * H * W;
  if (pix <= 0) return VSB_OK;
  im2col3x3_nhwc_kernel<<<(unsigned)pix, 128, 0, STREAM(stream)>>>((const bf16*)x, (bf16*)A, B, H, W, C);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_mask_dot_bf16(const void* up, const void* hyper, void* out, int B, long long P, int C, void* stream) {
  VSB_CHECK_ARG(up && hyper && out && C % 8 == 0, "vsb_mask_dot_bf16: bad args");
  const long long n = (long long)B * P;
  if (n <= 0) return VSB_OK;
  mask_dot_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM(stream)>>>((const bf16*)up, (const bf16*)hyper, (float*)out, B, P, C);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

// out [h,w] fp32, stats3 = (max, min, sum) of the written map; scratch >= 3*VSB_HEATMAP_MAX_BLOCKS floats
extern "C" int vsb_heatmap_bilinear_f32(const void* low, int LH, int LW, void* out, int h, int w, int do_clamp, void* scratch,
                                        void* stats3, void* stream) {
  VSB_CHECK_ARG(low && out && h > 0 && w > 0 && LH > 0 && LW > 0, "vsb_heatmap_bilinear_f32: bad args");
  VSB_CHECK_ARG((scratch != nullptr) == (stats3 != nullptr), "vsb_heatmap_bilinear_f32: scratch and stats3 go together");
  const long long n = (long long)h * w;
  long long blocks = (n + 256 * 8 - 1) / (256 * 8);
  if (blocks > VSB_HEATMAP_MAX_BLOCKS) blocks = VSB_HEATMAP_MAX_BLOCKS;
  if (blocks < 1) blocks = 1;
  heatmap_kernel<<<(unsigned)blocks, 256, 0, STREAM(stream)>>>((const float*)low, LH, LW, (float*)out, h, w, do_clamp, (float*)scratch);
  VSB_LAUNCH_CHECK();
  if (stats3) {
    stats_final_kernel<<<1, 256, 0, STREAM(stream)>>>((const float*)scratch, (int)blocks, (float*)stats3);
    VSB_LAUNCH_CHECK();
  }
  return VSB_OK;
}

extern "C" int vsb_rect_sums_f32(const void* hm, int h, int w, const void* rects, int nrects, const void* stats3, void* out_f64,
                                 void* scratch_f64, void* stream) {
  VSB_CHECK_ARG(hm && rects && stats3 && out_f64 && scratch_f64, "vsb_rect_sums_f32: null pointer (scratch = 64*nrects doubles)");
  if (nrects <= 0) return VSB_OK;
  dim3 grid(RECT_CHUNKS, nrects);
  rect_sums_partial_kernel<<<grid, 256, 0, STREAM(stream)>>>((const float*)hm, h, w, (const int*)rects, (const float*)stats3, (double*)scratch_f64);
  VSB_LAUNCH_CHECK();
  rect_sums_final_kernel<<<(nrects + 63) / 64, 64, 0, STREAM(stream)>>>((const double*)scratch_f64, nrects, (double*)out_f64);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_pack_detections_f32(const void* scores, const void* boxes, int n_crops, int P, void* rec, long long R, void* stream) {
  VSB_CHECK_ARG(scores && boxes && rec && P > 0 && R >= REC_PYR, "vsb_pack_detections_f32: bad args (record needs >= 76 floats)");
  VSB_CHECK_ARG(((uintptr_t)boxes & 15) == 0, "vsb_pack_detections_f32: boxes must be 16-byte aligned");
  if (n_crops <= 0) return VSB_OK;
  pack_detections_kernel<<<n_crops, 256, 0, STREAM(stream)>>>((const float*)scores, (const float*)boxes, P, (float*)rec, R);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_heat_pyramids_f32(const void* jobs_i32, int n_jobs, const void* rects_i32, const void* rect_job_i32, int total_rects,
                                     int LH, int LW, void* rec, long long R, void* scratch_stats_f32, void* scratch_rects_f64, void* stream) {
  VSB_CHECK_ARG(jobs_i32 && rec && scratch_stats_f32 && LH > 0 && LW > 0 && R >= REC_PYR, "vsb_heat_pyramids_f32: bad args");
  VSB_CHECK_ARG(total_rects == 0 || (rects_i32 && rect_job_i32 && scratch_rects_f64), "vsb_heat_pyramids_f32: rectangle tables missing");
  if (n_jobs <= 0) return VSB_OK;
  heat_stats_kernel<<<dim3(STAT_CHUNKS, n_jobs), 256, 0, STREAM(stream)>>>((const int*)jobs_i32, LH, LW, (float*)scratch_stats_f32);
  VSB_LAUNCH_CHECK();
  heat_stats_final_kernel<<<(n_jobs + 3) / 4, 128, 0, STREAM(stream)>>>((const int*)jobs_i32, n_jobs, (const float*)scratch_stats_f32,
                                                                        (float*)rec, R);
  VSB_LAUNCH_CHECK();
  if (total_rects > 0) {
    heat_rects_kernel<<<dim3(total_rects, RECT_CHUNKS), 256, 0, STREAM(stream)>>>((const int*)jobs_i32, (const int*)rects_i32,
                                                                                  (const int*)rect_job_i32, LH, LW, (const float*)rec, R,
                                                                                  (double*)scratch_rects_f64);
    VSB_LAUNCH_CHECK();
    heat_rects_final_kernel<<<(total_rects + 127) / 128, 128, 0, STREAM(stream)>>>((const int*)jobs_i32, (const int*)rect_job_i32,
                                                                                   total_rects, (const double*)scratch_rects_f64,
                                                                                   (float*)rec, R);
    VSB_LAUNCH_CHECK();
  }
  return VSB_OK;
}

extern "C" int vsb_copy2d_b16(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols, void* stream) {
  VSB_CHECK_ARG(src && dst && cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0, "vsb_copy2d_b16: cols/ld must be multiples of 8 elements");
  VSB_CHECK_ARG(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0, "vsb_copy2d_b16: 16-byte alignment required");
  const long long n = rows * (cols / 8);
  if (n <= 0) return VSB_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > vsb_num_sms() * 8) blocks = vsb_num_sms() * 8;
  copy2d_kernel<<<(unsigned)blocks, 256, 0, STREAM(stream)>>>((const uint4*)src, lds / 8, (uint4*)dst, ldd / 8, rows, cols / 8);
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}
