// Native runner for the Llama decoder stack on the fused-QKV cache (host code only: it sequences the kernels of this
// library).  One C call replaces 8 x n_layers Python->ctypes round trips; at decode (one token per step, every kernel a few
// microseconds) the Python wrappers, not the GPU, set the pace.
//
// Per layer (HF LlamaDecoderLayer, transformers/models/llama/modeling_llama.py; called through
// /root/reference/VisualSearch/model/llava/model/language_model/llava_llama.py:93-105 and
// /root/reference/LLaVA/llava/model/language_model/llava_search_llama.py:80-92):
//   h = RMSNorm(x) ; q|k|v = h Wqkv^T written straight into cache rows past..past+Tn ; RoPE in place ;
//   a = causal attention over cache rows 0..past+Tn ; x += a Wo^T ; h = RMSNorm(x) ; g = SwiGLU(h Wgu^T) ; x += g Wdown^T
#include "common.cuh"
#include "vstar_b200.h"

#include <math.h>

template <typename T>
int vsb_flash_attn_tc(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs, long long k_rs,
                      long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk, int D, int causal,
                      float scale, cudaStream_t stream);

// A/B and test switch: 0 (default) = vsb_llama_layers runs RoPE as its own kernel after the QKV projection, 1 = in the GEMM epilogue.
// The epilogue form must run 256-wide tiles (two heads each); the plain QKV GEMM runs 128-wide ones, and with the rope kernel after
// it the prefill step is ~5 % faster on H100 (DESIGN.md §6)
static int g_fuse_rope = 0;
extern "C" int vsb_llama_set_fuse_rope(int on) {
  g_fuse_rope = on ? 1 : 0;
  return VSB_OK;
}

#define VSB_TRY(call)          \
  do {                         \
    int _r = (call);           \
    if (_r != VSB_OK) return _r; \
  } while (0)

// the entry points of one element type: the same layer sequence runs on bf16 (VSM, default VQA engine) or f16 weights
template <typename T>
struct LayerOps;
template <>
struct LayerOps<bf16> {
  static constexpr auto gemm = vsb_gemm_bf16;
  static constexpr auto gemm_rowscale = vsb_gemm_rowscale_bf16;
  static constexpr auto gemm_qkv_rope = vsb_gemm_qkv_rope_bf16;
  static constexpr auto rowsq = vsb_rowsq_bf16;
  static constexpr auto rmsnorm = vsb_rmsnorm_bf16;
  static constexpr auto rope = vsb_rope_bf16;
  static constexpr auto flash_attn = vsb_flash_attn_bf16;
  static constexpr auto flash_attn_seg = vsb_flash_attn_seg_bf16;
  static constexpr auto attn_decode = vsb_attn_decode_bf16;
};
template <>
struct LayerOps<half> {
  static constexpr auto gemm = vsb_gemm_f16;
  static constexpr auto gemm_rowscale = vsb_gemm_rowscale_f16;
  static constexpr auto gemm_qkv_rope = vsb_gemm_qkv_rope_f16;
  static constexpr auto rowsq = vsb_rowsq_f16;
  static constexpr auto rmsnorm = vsb_rmsnorm_f16;
  static constexpr auto rope = vsb_rope_f16;
  static constexpr auto flash_attn = vsb_flash_attn_f16;
  static constexpr auto flash_attn_seg = vsb_flash_attn_seg_f16;
  static constexpr auto attn_decode = vsb_attn_decode_f16;
};

template <typename T>
int vsb_attn_chunk_paged_tc(const void* q, long long ldq, const CUtensorMap& tkv, long long row0, int d, void* o, long long ldo, int page_rows,
                            const void* page_table, int pt_ld, const void* seg, int S, int R, int H, int D, float scale, cudaStream_t stream);
int vsb_pool_map(CUtensorMap* map, const void* pool, long long rows, long long cols, int f16);
int vsb_attn_chunk_check(const void* q, long long ldq, void* o, long long ldo, int page_rows, const void* page_table, int pt_ld,
                         const void* seg, int S, int R, int H, int D);

int vsb_nf4_variant(int M);   // nf4.cu: 0 = the NF4 GEMM of M rows dequantises W and runs the tile kernels

// slot decode (vsb_llama_layers_slots): one new row per sequence, each at its own cache slot and length
struct SlotRows {
  const void* slot;   // int32 [B] cache slot of row b
  const void* len;    // int32 [B] rows already cached in that slot: the new row is written at slot*Tmax + len
  int max_len;        // >= every len[b]
  // paged cache (vsb_llama_layers_slots_paged), page_table NULL otherwise: `cache` is the pool [n_layers][n_pages][page_rows][2d]
  // of k|v rows, `slot` indexes the rows of page_table [*, pt_ld]
  const void* page_table = nullptr;
  int pt_ld = 0, page_rows = 0, n_pages = 0;
  // chunked prefill (vsb_llama_layers_chunked_paged): the last chunk_rows rows are prompt rows in n_seg segments (seg [3][n_seg])
  int chunk_rows = 0, n_seg = 0;
  const void* seg = nullptr;
};

template <typename T>
static int llama_layers(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int Tn, int past, void* cache, int Bc,
                        int Tmax, int d, int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin,
                        const void* positions, const void* k_start, int tail_rows, const void* q_seg, int seg_lo, int norm_folded,
                        void* scratch, void* deq_scratch, void* stream, const SlotRows* slots = nullptr) {
  using K = LayerOps<T>;
  VSB_CHECK_ARG(layers && x && cache && rope_cos && rope_sin && scratch, "vsb_llama_layers: null pointer");
  VSB_CHECK_ARG(n_layers > 0 && B > 0 && Tn > 0 && past >= 0 && d > 0 && H > 0 && inter > 0, "vsb_llama_layers: bad shape");
  VSB_CHECK_ARG(B <= Bc && past + Tn <= Tmax, "vsb_llama_layers: B=%d Tn=%d past=%d exceed the cache [%d, %d]", B, Tn, past, Bc, Tmax);
  VSB_CHECK_ARG(d % H == 0, "vsb_llama_layers: hidden %d not divisible by heads %d", d, H);
  VSB_CHECK_ARG(k_start == nullptr || Tn <= 4, "vsb_llama_layers: ragged batches (k_start) need Tn <= 4, got %d", Tn);
  VSB_CHECK_ARG(q_seg == nullptr || (k_start == nullptr && tail_rows == 0), "vsb_llama_layers: q_seg excludes k_start / tail_rows");
  if (slots) {
    VSB_CHECK_ARG(slots->slot && slots->len && positions, "vsb_llama_layers_slots: null slot / len / pos");
    VSB_CHECK_ARG(slots->max_len >= 0 && slots->max_len < Tmax, "vsb_llama_layers_slots: max_len %d outside the %d cache rows of a slot",
                  slots->max_len, Tmax);
  }
  // weight format: NF4 codes where the block scales are set, dense weights where they are NULL
  const bool nf4 = layers[0].wqkv_scales != nullptr;
  for (int li = 0; li < n_layers; ++li) {
    const vsb_llama_layer_t& L = layers[li];
    const int n = !!L.wqkv_scales + !!L.wo_scales + !!L.wgu_scales + !!L.wdown_scales;
    VSB_CHECK_ARG(n == (nf4 ? 4 : 0), "vsb_llama_layers: layer %d mixes NF4 and dense projections (a table is all one or the other)", li);
  }
  if (nf4) {
    VSB_CHECK_ARG(ElemT<T>::is_f16, "vsb_llama_layers: NF4 projections compute in fp16 (vsb_llama_layers_f16)");
    VSB_CHECK_ARG(!norm_folded && tail_rows == 0, "vsb_llama_layers: NF4 projections need norm_folded = 0 and tail_rows = 0");
    VSB_CHECK_ARG(deq_scratch, "vsb_llama_layers: NF4 projections need deq_scratch");
  }
  const int hd = d / H;
  const long long rows = (long long)B * Tn;
  const long long ld = 3LL * d;
  const float scale = 1.0f / sqrtf((float)hd);
  T* xb = reinterpret_cast<T*>(x);
  T* h = reinterpret_cast<T*>(scratch);                 // [rows, d]
  T* attn = h + rows * d;                               // [rows, d]
  T* gu = attn + rows * d;                              // [rows, inter]
  // tail mode: the caller consumes only the last `tail_rows` rows of every sequence (answer-predicting rows and the [LOC]
  // row of the guided search).  K/V of the last layer are needed by nobody else, so that layer runs its attention,
  // o-projection and MLP over B*tail rows only (same kernels, same per-row arithmetic => same values on those rows).
  const bool tail = tail_rows > 0 && 2 * tail_rows <= Tn && k_start == nullptr && slots == nullptr && (hd == 64 || hd == 128);
  // the projections of this call run on the wgmma tile kernels, whose epilogues alone fold RMSNorm and RoPE in (row counts
  // that take the skinny / weight-streaming decode kernels keep the separate RMSNorm and RoPE kernels)
  const bool tiles = nf4 ? vsb_nf4_variant((int)rows) == 0 : (rows > 16 || vsb_batch_invariant());
  // Folded RMSNorm (norm_folded: the caller multiplied ln1 into wqkv's and ln2 into wgu's columns): the QKV and gate|up GEMMs
  // read the un-normalised residual stream and scale their output rows by 1/rms in the epilogue; the o-proj and down-proj GEMMs
  // leave the per-row partial sums of squares of what they store.  Two kernels and ~0.3 GB of traffic less per layer at 64 crops.
  const bool fused = norm_folded && k_start == nullptr && d % 32 == 0 && tiles;
  const int sqc = d / 32;                                  // partial sums per row left by a d-wide producer GEMM
  float* sq_a = reinterpret_cast<float*>(h);              // [sqc][rows]  input of the next QKV GEMM   (h itself is unused when fused)
  float* sq_b = sq_a + (long long)sqc * rows;             // [sqc][rows]  input of the gate|up GEMM
  if (fused) {
    VSB_CHECK_ARG((long long)2 * sqc * rows * 4 <= rows * d * 2, "vsb_llama_layers: scratch too small for the row statistics");
    VSB_TRY(K::rowsq(xb, d, sq_a, (int)rows, d, stream));
  }
  // one tensor map over the whole pool serves the chunk attention of every layer
  CUtensorMap pool_map;
  if (slots && slots->chunk_rows) VSB_TRY(vsb_pool_map(&pool_map, cache, (long long)n_layers * slots->n_pages * slots->page_rows, 2LL * d, ElemT<T>::is_f16));
  // RoPE in the QKV epilogue (head_dim 128): q / k reach the cache already rotated
  const bool rope_fused = g_fuse_rope && hd == 128 && d % 256 == 0 && k_start == nullptr && slots == nullptr && tiles;

  // C [M, N] (leading dimension ldc) = epi(A W^T), A [M, Kd] with leading dimension Kd, plus C itself when `accumulate` (the
  // residual stream).  NF4 W (scales set): vsb_gemm_nf4.  Dense W: the tile / skinny GEMM, or its row-scale form when the folded
  // norm's row statistics go in (sq_in, sq_chunks partial sums per row) or out (sq_out), both [chunks][M].
  auto proj = [&](const void* A, const void* W, const void* scales, void* C, long long ldc, long long M, int N, int Kd, bool accumulate,
                  int epi, int rows_per_group, long long group_stride, long long group_offset, const float* sq_in, int sq_chunks,
                  float* sq_out) -> int {
    const void* res = accumulate ? C : nullptr;
    const long long ldr = accumulate ? ldc : 0;
    if (scales)
      return vsb_gemm_nf4(A, Kd, W, scales, C, ldc, (int)M, N, Kd, nullptr, res, ldr, epi, 0, rows_per_group, group_stride, group_offset,
                          deq_scratch, stream);
    if (sq_in || sq_out)
      return K::gemm_rowscale(A, Kd, W, Kd, C, ldc, (int)M, N, Kd, nullptr, res, ldr, epi, rows_per_group, group_stride, group_offset, sq_in,
                              sq_chunks, rms_eps, sq_out, M, stream);
    return K::gemm(A, Kd, W, Kd, C, ldc, (int)M, N, Kd, nullptr, res, ldr, epi, 0, rows_per_group, group_stride, group_offset, stream);
  };
  // x += a Wo^T ; h = RMSNorm(x) ; g = SwiGLU(h Wgu^T) ; x += g Wdown^T over the R rows of X [R, d] whose attention output is in
  // attn.  Folded norms: the o-proj leaves the row statistics gate|up reads, and down-proj leaves them in sq_out (NULL: nowhere).
  auto post_attention = [&](const vsb_llama_layer_t& L, T* X, long long R, float* sq_out) -> int {
    VSB_TRY(proj(attn, L.wo, L.wo_scales, X, d, R, d, d, true, VSB_EPI_NONE, 0, 0, 0, nullptr, 0, fused ? sq_b : nullptr));
    if (!fused) VSB_TRY(K::rmsnorm(X, d, L.ln2, h, d, (int)R, d, rms_eps, stream));
    VSB_TRY(proj(fused ? X : h, L.wgu, L.wgu_scales, gu, inter, R, 2 * inter, d, false, VSB_EPI_SWIGLU, 0, 0, 0, fused ? sq_b : nullptr,
                 sqc, nullptr));
    return proj(gu, L.wdown, L.wdown_scales, X, d, R, d, inter, true, VSB_EPI_NONE, 0, 0, 0, nullptr, 0, sq_out);
  };

  for (int li = 0; li < n_layers; ++li) {
    const vsb_llama_layer_t& L = layers[li];
    T* cl = reinterpret_cast<T*>(cache) + (long long)li * Bc * Tmax * ld;       // [Bc*Tmax, 3d]
    if (!fused) VSB_TRY(K::rmsnorm(xb, d, L.ln1, h, d, (int)rows, d, rms_eps, stream));
    const T* qkv_in = fused ? xb : h;
    const float* sq_in = fused ? sq_a : nullptr;
    const int sq_in_chunks = !fused ? 0 : li == 0 ? 1 : sqc;   // layer 0: one full-row sum from K::rowsq
    if (slots) {
      // q|k|v into scratch, then rotated and scattered to each row's own cache row; attention over each row's own keys
      T* qkv = gu + rows * inter;                                                      // [B, 3d]
      VSB_TRY(proj(qkv_in, L.wqkv, L.wqkv_scales, qkv, ld, rows, 3 * d, d, false, VSB_EPI_NONE, 0, 0, 0, sq_in, sq_in_chunks, nullptr));
      const int dt = ElemT<T>::is_f16 ? VSB_DTYPE_F16 : VSB_DTYPE_BF16;
      if (slots->page_table) {
        // q rotated in place in scratch, k|v to the row's page; attention reads q there and k|v through the page table
        const long long kv = 2LL * d, page = (long long)slots->page_rows * kv;
        T* pl = reinterpret_cast<T*>(cache) + (long long)li * slots->n_pages * page;  // [n_pages, page_rows, 2d]
        // chunk rows: row i of a segment is a row with len = pos = lo + i, so the same scatter places it
        const int nd = B - slots->chunk_rows;                                         // decode rows, first
        VSB_TRY(vsb_rope_scatter_paged(qkv, ld, B, H, hd, pl, page, kv, slots->page_rows, slots->page_table, slots->pt_ld, slots->slot, slots->len,
                                       positions, rope_cos, rope_sin, dt, stream));
        if (nd > 0)
          VSB_TRY(vsb_attn_decode_paged(qkv, ld, pl, pl + d, attn, d, page, kv, slots->page_rows, slots->page_table, slots->pt_ld, nd, H, hd,
                                        scale, slots->slot, slots->len, slots->max_len, dt, stream));
        if (slots->chunk_rows)
          VSB_TRY(vsb_attn_chunk_paged_tc<T>(qkv + nd * ld, ld, pool_map, (long long)li * slots->n_pages * slots->page_rows, d, attn + (long long)nd * d,
                                             d, slots->page_rows, slots->page_table, slots->pt_ld, slots->seg, slots->n_seg, slots->chunk_rows, H,
                                             hd, scale, reinterpret_cast<cudaStream_t>(stream)));
      } else {
        VSB_TRY(vsb_rope_scatter(qkv, ld, B, H, hd, cl, ld, Tmax, slots->slot, slots->len, positions, rope_cos, rope_sin, dt, stream));
        VSB_TRY(vsb_attn_decode_slots(cl, cl + d, cl + 2 * d, attn, (long long)Tmax * ld, ld, d, B, H, hd, scale, slots->slot, slots->len,
                                      slots->max_len, dt, stream));
      }
      VSB_TRY(post_attention(L, xb, rows, fused ? sq_a : nullptr));
      continue;
    }
    if (rope_fused) {
      const void* wqkv = L.wqkv;
      if (nf4) {                                               // the RoPE epilogue has no NF4 form: it runs on deq(wqkv)
        VSB_TRY(vsb_nf4_dequant(L.wqkv, L.wqkv_scales, 3 * d, d, deq_scratch, d, stream));
        wqkv = deq_scratch;
      }
      VSB_TRY(K::gemm_qkv_rope(qkv_in, d, wqkv, d, cl, ld, (int)rows, 3 * d, d, Tn, Tmax, past, sq_in, sq_in_chunks, rms_eps, rows, rope_cos,
                               rope_sin, positions, Tn, past, hd, stream));
    } else {
      VSB_TRY(proj(qkv_in, L.wqkv, L.wqkv_scales, cl, ld, rows, 3 * d, d, false, VSB_EPI_NONE, Tn, Tmax, past, sq_in, sq_in_chunks, nullptr));
      VSB_TRY(K::rope(cl, ld, (int)rows, Tn, H, hd, past, rope_cos, rope_sin, positions, Tmax, past, stream));
    }
    if (tail && li == n_layers - 1) {
      const long long trows = (long long)B * tail_rows;
      T* xt = attn + trows * d;                                                     // compact copy of the tail rows of x
      const int q0 = past + Tn - tail_rows;
      VSB_TRY(vsb_flash_attn_tc<T>(cl + (long long)q0 * ld, cl + d, cl + 2 * d, attn, (long long)Tmax * ld, ld, (long long)Tmax * ld, ld,
                                (long long)Tmax * ld, ld, (long long)tail_rows * d, d, B, H, tail_rows, past + Tn, hd, 1, scale,
                                reinterpret_cast<cudaStream_t>(stream)));
      VSB_TRY(vsb_copy2d_b16(xb + (long long)(Tn - tail_rows) * d, (long long)Tn * d, xt, (long long)tail_rows * d, B, tail_rows * d, stream));
      // compact tail rows: same kernels on trows rows (sq_b is indexed by compact row, leading dimension trows)
      VSB_TRY(post_attention(L, xt, trows, nullptr));
      VSB_TRY(vsb_copy2d_b16(xt, (long long)tail_rows * d, xb + (long long)(Tn - tail_rows) * d, (long long)Tn * d, B, tail_rows * d, stream));
      break;
    }
    if (q_seg != nullptr)
      VSB_TRY(K::flash_attn_seg(cl + (long long)past * ld, cl + d, cl + 2 * d, attn, (long long)Tmax * ld, ld, (long long)Tmax * ld, ld,
                                      (long long)Tmax * ld, ld, (long long)Tn * d, d, B, H, Tn, past + Tn, hd, scale, q_seg, seg_lo, stream));
    else if (k_start != nullptr)
      VSB_TRY(K::attn_decode(cl + (long long)past * ld, cl + d, cl + 2 * d, attn, (long long)Tmax * ld, ld, (long long)Tmax * ld, ld,
                                   (long long)Tmax * ld, ld, (long long)Tn * d, d, B, H, Tn, past + Tn, hd, 1, scale, k_start, stream));
    else
      VSB_TRY(K::flash_attn(cl + (long long)past * ld, cl + d, cl + 2 * d, attn, (long long)Tmax * ld, ld, (long long)Tmax * ld, ld,
                                  (long long)Tmax * ld, ld, (long long)Tn * d, d, B, H, Tn, past + Tn, hd, 1, scale, stream));
    // the down projection leaves the row statistics the NEXT layer's QKV GEMM needs (nobody reads them after the last layer)
    VSB_TRY(post_attention(L, xb, rows, fused ? sq_a : nullptr));
  }
  return VSB_OK;
}

extern "C" int vsb_llama_layers(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int Tn, int past, void* cache, int Bc,
                                int Tmax, int d, int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin,
                                const void* positions, const void* k_start, int tail_rows, const void* q_seg, int seg_lo, int norm_folded,
                                void* scratch, void* deq_scratch, void* stream) {
  return llama_layers<bf16>(layers, n_layers, x, B, Tn, past, cache, Bc, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, positions, k_start,
                            tail_rows, q_seg, seg_lo, norm_folded, scratch, deq_scratch, stream);
}
extern "C" int vsb_llama_layers_f16(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int Tn, int past, void* cache, int Bc,
                                    int Tmax, int d, int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin,
                                    const void* positions, const void* k_start, int tail_rows, const void* q_seg, int seg_lo, int norm_folded,
                                    void* scratch, void* deq_scratch, void* stream) {
  return llama_layers<half>(layers, n_layers, x, B, Tn, past, cache, Bc, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, positions, k_start,
                            tail_rows, q_seg, seg_lo, norm_folded, scratch, deq_scratch, stream);
}

// Slot decode: one new token per sequence, every sequence at its own cache slot and length (a decode batch that admits a new
// sequence whenever another one ends).  Same per-layer sequence as vsb_llama_layers with Tn = 1, except that the QKV projection
// goes to scratch and vsb_rope_scatter / vsb_attn_decode_slots place and read each row's keys.
extern "C" int vsb_llama_layers_slots(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, void* cache, int Bc, int Tmax, int d,
                                      int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin, const void* slot_i32,
                                      const void* len_i32, const void* pos_i32, int max_len, int norm_folded, void* scratch,
                                      void* deq_scratch, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_llama_layers_slots: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)", dtype);
  const SlotRows s{slot_i32, len_i32, max_len};
  if (dtype == VSB_DTYPE_F16)
    return llama_layers<half>(layers, n_layers, x, B, 1, 0, cache, Bc, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr, 0,
                              nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
  return llama_layers<bf16>(layers, n_layers, x, B, 1, 0, cache, Bc, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr, 0,
                            nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
}

// Paged slot decode: vsb_llama_layers_slots on a pool of k|v pages instead of one [Tmax, 3d] slot per sequence.  Row b's new q is
// rotated in place in scratch, its k|v go to row len[b] of the pages page_table[slot[b]] lists (vsb_rope_scatter_paged), and
// vsb_attn_decode_paged reads its keys through the same table.  Every other kernel of the layer is the slot runner's.
extern "C" int vsb_llama_layers_slots_paged(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, void* pool, int n_pages, int page_rows,
                                            const void* page_table_i32, int pt_ld, int d, int H, int inter, float rms_eps, const void* rope_cos,
                                            const void* rope_sin, const void* slot_i32, const void* len_i32, const void* pos_i32, int max_len,
                                            int norm_folded, void* scratch, void* deq_scratch, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_llama_layers_slots_paged: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)",
                dtype);
  VSB_CHECK_ARG(page_table_i32 && n_pages > 0 && pt_ld > 0, "vsb_llama_layers_slots_paged: null page table or empty pool");
  VSB_CHECK_ARG(page_rows >= 16 && (page_rows & (page_rows - 1)) == 0 && (long long)pt_ld * page_rows < (1LL << 30),
                "vsb_llama_layers_slots_paged: page_rows %d is not a power of two >= 16", page_rows);
  SlotRows s{slot_i32, len_i32, max_len};
  s.page_table = page_table_i32;
  s.pt_ld = pt_ld;
  s.page_rows = page_rows;
  s.n_pages = n_pages;
  // the cache-shape checks of the runner see B sequences of pt_ld * page_rows rows
  const int Tmax = pt_ld * page_rows;
  if (dtype == VSB_DTYPE_F16)
    return llama_layers<half>(layers, n_layers, x, B, 1, 0, pool, B, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr, 0,
                              nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
  return llama_layers<bf16>(layers, n_layers, x, B, 1, 0, pool, B, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr, 0,
                            nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
}

// Chunked prefill: vsb_llama_layers_slots_paged on B decode rows followed by R prompt rows in S segments (x [B + R, d]).  Every
// kernel runs on all B + R rows but attention: vsb_attn_decode_paged for the decode rows, vsb_attn_chunk_paged for the chunk rows.
extern "C" int vsb_llama_layers_chunked_paged(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int R, void* pool, int n_pages,
                                              int page_rows, const void* page_table_i32, int pt_ld, int d, int H, int inter, float rms_eps,
                                              const void* rope_cos, const void* rope_sin, const void* slot_i32, const void* len_i32,
                                              const void* pos_i32, int max_len, const void* seg_i32, int S, int norm_folded, void* scratch,
                                              void* deq_scratch, int dtype, void* stream) {
  VSB_CHECK_ARG(dtype == VSB_DTYPE_BF16 || dtype == VSB_DTYPE_F16, "vsb_llama_layers_chunked_paged: dtype %d (VSB_DTYPE_BF16 / VSB_DTYPE_F16)",
                dtype);
  VSB_CHECK_ARG(page_table_i32 && n_pages > 0 && pt_ld > 0 && B >= 0 && H > 0 && d % H == 0,
                "vsb_llama_layers_chunked_paged: null page table, empty pool or bad shape");
  VSB_CHECK_ARG((long long)n_layers * n_pages * page_rows < (1LL << 31), "vsb_llama_layers_chunked_paged: pool of %d x %d x %d rows", n_layers,
                n_pages, page_rows);
  // the chunk kernel's refusals before the first launch of the stack (its q / o are the runner's scratch rows)
  const long long rows = (long long)B + R;
  const void* q = reinterpret_cast<const char*>(scratch) + rows * (2LL * d + inter) * 2 + (long long)B * 3 * d * 2;
  VSB_TRY(vsb_attn_chunk_check(q, 3LL * d, scratch, d, page_rows, page_table_i32, pt_ld, seg_i32, S, R, H, d / H));
  SlotRows s{slot_i32, len_i32, max_len};
  s.page_table = page_table_i32;
  s.pt_ld = pt_ld;
  s.page_rows = page_rows;
  s.n_pages = n_pages;
  s.chunk_rows = R;
  s.n_seg = S;
  s.seg = seg_i32;
  const int Tmax = pt_ld * page_rows;
  if (dtype == VSB_DTYPE_F16)
    return llama_layers<half>(layers, n_layers, x, (int)rows, 1, 0, pool, (int)rows, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr,
                              0, nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
  return llama_layers<bf16>(layers, n_layers, x, (int)rows, 1, 0, pool, (int)rows, Tmax, d, H, inter, rms_eps, rope_cos, rope_sin, pos_i32, nullptr,
                            0, nullptr, 0, norm_folded, scratch, deq_scratch, stream, &s);
}
