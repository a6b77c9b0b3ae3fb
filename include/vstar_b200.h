/* vstar_b200 C-ABI — the drop-in boundary of the H100-native V* (SEAL) visual-search hot path.
 *
 * The reference (penghao-wu/vstar) is pure Python and has no FFI layer of its own: the boundary it
 * exposes is the Python API of visual_search.py / VSM.py (SURVEY.md §8b), mirrored by the host code in
 * vstar_b200/.  Underneath that mirror every arithmetic op of the path is one of the entry points
 * below: plain C, raw DEVICE pointers + sizes + a cudaStream_t passed as void*, no torch types, no
 * allocation inside, no global state except a TMA-descriptor cache.  Each entry point cites the
 * reference op site(s) (file:line) it replaces.
 *
 * Return value: 0 on success, negative on error (VSB_ERR_*); vsb_last_error() gives the message.
 * All matrices are row-major; "ld*" are leading dimensions in ELEMENTS; bf16 = __nv_bfloat16, f16 = IEEE half.
 *
 * Every entry point the SEAL VQA LLM reaches has an _f16 twin with the _bf16 signature: same kernels instantiated for f16
 * operands and outputs (fp32 accumulation and statistics either way), so that model runs in fp16 like the reference
 * (LLaVA/llava/model/builder.py:43).  Pure 2-byte copies (gather_rows, patchify, copy2d) serve both types as they are.
 */
#ifndef VSTAR_B200_H_
#define VSTAR_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define VSB_EPI_NONE 0
#define VSB_EPI_QUICK_GELU 1 /* x*sigmoid(1.702x): CLIP / OWL-ViT MLP (transformers/activations.py:117-123) */
#define VSB_EPI_GELU 2       /* exact erf GELU: OWL box head, SAM upscaling */
#define VSB_EPI_RELU 3       /* SAM transformer MLP, text_hidden_fcs, hyper-network MLPs */
#define VSB_EPI_SWIGLU 4     /* silu(gate)*up with gate/up rows interleaved in W (Llama MLP) */

#define VSB_DTYPE_BF16 0 /* logit_dtype of vsb_sample_rows_f32: the engine dtype the logits are rounded to */
#define VSB_DTYPE_F16 1

#define VSB_HEATMAP_MAX_BLOCKS 1184 /* blocks of the heat-map reduction (fixed: its summation order does not depend on the GPU) */

const char* vsb_last_error(void);
int vsb_version(void);
/* 1: kernels are chosen independently of the number of rows in a call (no skinny-GEMM / row-RMSNorm shortcuts), so a crop's result
 * does not depend on how many other crops share its batch - required for identical search trajectories under speculative
 * batching and frontier sharding (SURVEY.md section 8e).  0 (default): fastest kernel per shape (decode paths). */
int vsb_set_batch_invariant(int on);

/* C[M,N] = epi(A[M,K] . W[N,K]^T + bias[N]) (+ residual[M,N]); TMA + wgmma GEMM, bf16 operands, fp32
 * accumulate.  out_fp32: C/residual element type (0 = bf16, 1 = fp32).  Output-row remap (rows_per_group > 0):
 * row m -> (m / rows_per_group) * group_stride + group_offset + m % rows_per_group (used to scatter the 256
 * projected CLIP rows of each crop straight into the LLM input buffer; llava_arch.py:185-208).
 * Replaces every nn.Linear / conv-as-GEMM on the path:
 *   VisualSearch/model/llava/model/llava_arch.py:93-96 (mm_projector); HF LlamaModel q/k/v/o/gate/up/down and
 *   lm_head via llava_llama.py:93-105; HF CLIP/OWL-ViT patch-embed + encoder linears via clip_encoder.py:53-57
 *   and owlvit.py:121-126; VSM.py:117-140 (text_hidden_fcs), :88 (visual_projection); owlvit.py:79-119 heads;
 *   segment_anything/modeling/transformer.py:205-242, mask_decoder.py:15-27,:191-213. */
int vsb_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                  const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                  long long group_stride, long long group_offset, void* stream);
/* f16 twin of vsb_gemm_bf16 (A, W, bias and a non-fp32 C / residual are f16) */
int vsb_gemm_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                 const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                 long long group_stride, long long group_offset, void* stream);
/* vsb_gemm_bf16 with HF LlamaRMSNorm (modeling_llama.py:53-67) FOLDED IN; the norm weight must already be multiplied into W's columns.
 * rowsq_in != NULL: output row m is scaled by rsqrt(sum_c rowsq_in[c*sq_ld + m] / K + eps) before bias / activation, i.e. A is the
 * UN-normalised residual stream and 1/rms is applied in the epilogue (no norm kernel, no normalised copy of the activations).
 * rowsq_out != NULL (bf16 output, N % 32 == 0): also writes the sum of squares of every stored 32-value chunk,
 * rowsq_out[(n/32)*sq_ld + row], which the next folded GEMM consumes with sq_in_chunks = N/32.  wgmma tile kernels for any M. */
int vsb_gemm_rowscale_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                           const void* bias, const void* residual, long long ldr, int epilogue, int rows_per_group, long long group_stride,
                           long long group_offset, const void* rowsq_in, int sq_in_chunks, float eps, void* rowsq_out, long long sq_ld,
                           void* stream);
/* f16 twin of vsb_gemm_rowscale_bf16 */
int vsb_gemm_rowscale_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                          const void* bias, const void* residual, long long ldr, int epilogue, int rows_per_group, long long group_stride,
                          long long group_offset, const void* rowsq_in, int sq_in_chunks, float eps, void* rowsq_out, long long sq_ld,
                          void* stream);
/* Fused QKV projection of a Llama layer (HF LlamaAttention q/k/v_proj + apply_rotary_pos_emb, modeling_llama.py:138-168, :199-221):
 * C = [q | k | v] = A . W^T, optional folded RMSNorm (rowsq_in as above), and rotate-half RoPE applied by the epilogue to the q and k
 * thirds (head_dim 128; cos/sin tables bf16 [max_pos, 64]; position of row m = positions[m] or pos0 + m % T), so q / k land in the KV
 * cache already rotated.  Bit-identical to vsb_gemm_bf16 followed by vsb_rope_bf16. */
int vsb_gemm_qkv_rope_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                           int rows_per_group, long long group_stride, long long group_offset, const void* rowsq_in, int sq_in_chunks,
                           float eps, long long sq_ld, const void* cos_table, const void* sin_table, const void* positions, int T, int pos0,
                           int head_dim, void* stream);
/* f16 twin of vsb_gemm_qkv_rope_bf16 (f16 cos/sin tables); bit-identical to vsb_gemm_f16 followed by vsb_rope_f16 */
int vsb_gemm_qkv_rope_f16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                          int rows_per_group, long long group_stride, long long group_offset, const void* rowsq_in, int sq_in_chunks,
                          float eps, long long sq_ld, const void* cos_table, const void* sin_table, const void* positions, int T, int pos0,
                          int head_dim, void* stream);
/* 1: vsb_llama_layers applies RoPE in the QKV GEMM epilogue (head_dim 128); 0 (default): separate vsb_rope_bf16 launch */
int vsb_llama_set_fuse_rope(int on);
/* per-row sum of squares (fp32) of a bf16 matrix: the first rowsq_in of a chain of folded GEMMs (sq_in_chunks = 1) */
int vsb_rowsq_bf16(const void* x, long long ldx, void* out_f32, int rows, int cols, void* stream);
/* f16 twin of vsb_rowsq_bf16 */
int vsb_rowsq_f16(const void* x, long long ldx, void* out_f32, int rows, int cols, void* stream);
/* CUDA-event profiling of every vsb_gemm_bf16 launch (bench.py's roofline leg): begin clears the record; end synchronises
 * and returns the summed algorithmic flops (2*M*N*K), the summed event durations in ms and the launch count. */
int vsb_gemm_profile_begin(void);
int vsb_gemm_profile_end(double* flops, double* ms, long long* launches);
/* testing / tuning hooks: force the kernel variant (1 = CUDA-core skinny kernel for M <= 8, 2 = mma.sync skinny kernel for M <= 16,
 * 32/64/128/256 = wgmma tile width, 0 = auto) and the CTA count (0 = #SMs); tile-rasterisation band height in m-blocks (0 = auto) */
int vsb_gemm_set_tuning(int force_bn, int max_ctas);
int vsb_gemm_set_group_m(int group_m);
/* L2 eviction hints of the tile kernel on large GEMMs (M, N >= 512, K >= 1024), bit mask: 1 = A tiles evict_last,
 * 2 = W tiles evict_first, 8 = W tiles evict_last, 4 = streaming (.cs) output stores; 0 = none (default). */
int vsb_gemm_set_l2_hints(int on);

/* nn.LayerNorm over the last dim (fp32 stats), optional fused activation (VSB_EPI_NONE / VSB_EPI_GELU).
 * HF CLIP/OWL layer_norm1/2, pre/post layernorm; SAM norm1-4, norm_final_attn; LayerNorm2d in NHWC (common.py:31-43). */
int vsb_layernorm_bf16(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int rows, int cols,
                       float eps, int act, void* stream);
/* f16 twin of vsb_layernorm_bf16 */
int vsb_layernorm_f16(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int rows, int cols,
                      float eps, int act, void* stream);
/* HF LlamaRMSNorm (transformers/models/llama/modeling_llama.py:53-67): y = w * bf16(x * rsqrt(mean(x^2)+eps)). */
int vsb_rmsnorm_bf16(const void* x, long long ldx, const void* w, void* y, long long ldy, int rows, int cols, float eps, void* stream);
/* f16 twin of vsb_rmsnorm_bf16: y = w * f16(x * rsqrt(mean(x^2)+eps)), as HF LlamaRMSNorm in fp16 */
int vsb_rmsnorm_f16(const void* x, long long ldx, const void* w, void* y, long long ldy, int rows, int cols, float eps, void* stream);
/* rotate-half RoPE in place on the q and k thirds of a fused qkv buffer [.., 3*H*D]
 * (modeling_llama.py:117-168); cos/sin tables bf16 [max_pos, D/2]; position = positions[r] or pos0 + r % T;
 * logical row r is stored at physical row (r / T) * group_stride + group_offset + r % T (KV-cache layout). */
int vsb_rope_bf16(void* qkv, long long ld, int rows, int T, int H, int D, int pos0, const void* cos_table, const void* sin_table,
                  const void* positions, long long group_stride, long long group_offset, void* stream);
/* f16 twin of vsb_rope_bf16 (f16 tables; f16 rounding of each product and of the sum, as HF in fp16) */
int vsb_rope_f16(void* qkv, long long ld, int rows, int T, int H, int D, int pos0, const void* cos_table, const void* sin_table,
                 const void* positions, long long group_stride, long long group_offset, void* stream);
/* embed_tokens lookup for the text slots of the spliced sequence (llava_arch.py:185-208, :235-251);
 * ids int64 [B,L] with the image placeholder at img_pos; out [B, L-1+n_img, d]. */
int vsb_embed_splice_bf16(const void* ids, const void* table, void* out, int B, int L, int img_pos, int n_img, int d, int vocab, void* stream);
int vsb_gather_rows_bf16(const void* idx_i64, const void* table, long long ldt, void* out, long long ldo, int n, int d,
                         long long nrows_table, void* stream);
/* im2col for the stride==kernel patch-embedding conv (HF CLIPVisionEmbeddings / OwlViTVisionEmbeddings). */
int vsb_patchify_bf16(const void* pixels, void* A, int B, int S, int P, int Kpad, void* stream);
/* x[:,0] = cls + pos[0]; x[:,1:] += pos[1:] */
int vsb_vit_add_pos_bf16(void* x, const void* cls, const void* pos, int B, int S, int C, void* stream);
/* f16 twin of vsb_vit_add_pos_bf16 */
int vsb_vit_add_pos_f16(void* x, const void* cls, const void* pos, int B, int S, int C, void* stream);
/* OwlViT.get_visual_embs tail (owlvit.py:128-138): LN2(LN1(x[:,1:]) * LN1(x[:,:1])). */
int vsb_owl_merge_bf16(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, void* y, int B, int S, int C,
                       float eps, void* stream);
int vsb_add_rows_bf16(const void* a, const void* b, void* y, long long rows, int cols, long long bmod, void* stream);
/* f16 twin of vsb_add_rows_bf16 */
int vsb_add_rows_f16(const void* a, const void* b, void* y, long long rows, int cols, long long bmod, void* stream);
int vsb_cast_f32_bf16(const void* x, void* y, long long n, void* stream);
/* f16 twin of vsb_cast_f32_bf16 (the reference's .half() of fp32 pixels) */
int vsb_cast_f32_f16(const void* x, void* y, long long n, void* stream);
/* Greedy token of every row of fp32 logits [rows, n]: torch.argmax's index (the first maximum; NaN counts as the largest value,
 * the first NaN wins) and its value */
int vsb_argmax_rows_f32(const void* x, long long ld, int rows, int n, void* idx_i32, void* val_f32, void* stream);
/* Sampled next token of every row of fp32 logits [rows, n] (HF `sample()` with TemperatureLogitsWarper, TopKLogitsWarper,
 * TopPLogitsWarper and multinomial(softmax), as transformers 4.31 runs them for free_form_inference(temperature > 0)).  Per row:
 * v = dtype(float(dtype(x)) / temperature) with dtype = logit_dtype (VSB_DTYPE_BF16 / VSB_DTYPE_F16: the reference's logits
 * are the lm_head output in the model dtype); top_k > 0 keeps every v >= the k-th largest (ties kept), 0 disables it;
 * top_p < 1 keeps, in descending order, each position whose probability mass at or after it exceeds 1 - top_p (the largest
 * always kept), 1 disables it; probabilities in fp64 from exp(v - max).  The token is drawn by inverse CDF over the kept tokens
 * (descending v, ties by ascending id) at u = Philox4x32-10(key = seeds_i64[row], counter = (step, 0, 0, 0)), 53 bits, so it
 * depends only on the row's logits, its seed and step.  seeds_i64: device int64 [rows]; idx_i32: device int32 [rows]. */
int vsb_sample_rows_f32(const void* logits, long long ld, int rows, int n, float temperature, int top_k, float top_p, int logit_dtype,
                        const void* seeds_i64, int step, void* idx_i32, void* stream);
/* vsb_sample_rows_f32 with every row's own settings (a decode stream, each request at its own step): temperature_f32 (> 0),
 * top_k_i32 (0 = off), top_p_f32 (1 = off), seeds_i64 and steps_i32 are device arrays [rows]; the row's token is the one
 * vsb_sample_rows_f32 draws for the same logits, settings, seed and step.  The caller validates the settings. */
int vsb_sample_rows_var_f32(const void* logits, long long ld, int rows, int n, const void* temperature_f32, const void* top_k_i32,
                            const void* top_p_f32, int logit_dtype, const void* seeds_i64, const void* steps_i32, void* idx_i32,
                            void* stream);
/* per-row negative log-likelihood of labels under softmax(logits) — option scoring of the SEAL VQA LLM
 * (CrossEntropyLoss, /root/reference/vstar_bench_eval.py:154-159) */
int vsb_nll_rows_f32(const void* logits, long long ld, int rows, int n, const void* labels_i64, void* out_f32, void* stream);
int vsb_copy2d_b16(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols, void* stream);

/* Beam search of the SEAL VQA LLM (HF `beam_search` of transformers 4.31 for free_form_inference(num_beams = k),
 * /root/reference/vstar_bench_eval.py:91-103).  Candidates of one step for `requests` requests of k_in rows each (1 on the first
 * step, k afterwards): rows_i32 [requests, k_in] are the rows of the fp32 logits [*, V] (cache-slot order) that hold the
 * request's beams in beam order, scores_f32 [requests, k_in] their running scores.  Per row, logp = dtype(x - max - log sum
 * exp(x - max)) of x = float(dtype(logit)) (sum and difference in fp64, rounded once to logit_dtype), candidate score
 * float(logp) + beam score in fp32.  Output per request: the 2k largest candidate scores over k_in * V, descending, ties by
 * ascending beam * V + token: out_score_f32, out_token_i32, out_beam_i32 [requests, 2k] (device).  1 <= k <= VSB_BEAM_MAX. */
#define VSB_BEAM_MAX 16
int vsb_beam_candidates_f32(const void* logits, long long ld, int V, int requests, int k_in, int k, const void* rows_i32,
                            const void* scores_f32, int logit_dtype, void* out_score_f32, void* out_token_i32, void* out_beam_i32,
                            void* stream);
/* Beam reordering of the fused-QKV cache: for every layer l < layers and every pair p, rows [lo, hi) of slot
 * pairs_i32[2p] are copied bit-exactly to slot pairs_i32[2p+1] (element (l, slot, row, c) at cache + l*layer_stride +
 * slot*slot_stride + row*row_stride + c, c < row_elems; 2-byte elements).  pairs_i32 is a HOST array of npairs (src, dst)
 * pairs, at most VSB_COPY_ROWS_MAX_PAIRS; a slot that is both a source and a destination, a destination named twice or a slot
 * outside [0, slots) is refused with VSB_ERR_ARG.  One launch. */
#define VSB_COPY_ROWS_MAX_PAIRS 256
int vsb_copy_cache_rows_b16(void* cache, int layers, long long layer_stride, int slots, long long slot_stride, long long row_stride,
                            int row_elems, const int* pairs_i32, int npairs, int lo, int hi, void* stream);
/* vsb_copy_cache_rows_b16 with a row range per pair: quads_i32 is a HOST array of npairs (src, dst, lo, hi), rows [lo, hi) of
 * slot src copied to slot dst for every layer.  Refused with VSB_ERR_ARG before any launch: a slot that is both a source and a
 * destination, a destination named twice, a slot outside [0, slots), lo > hi or a range past the slot; slots <= 65536.
 * One launch. */
int vsb_copy_slot_rows_b16(void* cache, int layers, long long layer_stride, int slots, long long slot_stride, long long row_stride,
                           int row_elems, const int* quads_i32, int npairs, void* stream);

/* The whole Llama decoder stack over Tn new rows per sequence, in place on the residual stream x [B*Tn, d] bf16
 * (HF LlamaModel layers as called from llava_llama.py:93-105 / llava_search_llama.py:80-92).  Fused q|k|v rows live in
 * cache [n_layers][Bc][Tmax][3d] at positions past..past+Tn; weights: wqkv [3d,d] (q|k|v rows), wo [d,d], wgu [2*inter,d]
 * with gate/up rows interleaved, wdown [d,inter], ln1/ln2 [d]; rope tables bf16 [max_pos, head_dim/2]; scratch: bf16
 * B*Tn*(2d+inter) elements.  Ragged batches (continuous-batched decode): sequences are LEFT-padded in the cache so that
 * they all end at row past+Tn; positions int32 [B*Tn] gives each new row its RoPE position and k_start int32 [B] the first
 * cache row of each sequence (requires Tn <= 4); both NULL for the aligned case.  tail_rows > 0: the caller will read only
 * the last tail_rows rows of every sequence, so the LAST layer runs attention / o-proj / MLP on those rows only (all other
 * rows of x are left at their layer n-1 value); 0 = every row.  q_seg int32 [B*Tn] (with positions): the new rows are several
 * CONTINUATIONS of the cached prefix appended back to back (answer options, vstar_bench_eval.py:127-163): row r attends the
 * prefix keys [0, seg_lo) and its own continuation from key q_seg[r] on (vsb_flash_attn_seg_bf16).  norm_folded != 0: the caller
 * has multiplied ln1 into wqkv's columns and ln2 into wgu's (ln1 / ln2 then hold ones): the QKV and gate|up GEMMs take the
 * un-normalised residual stream and apply 1/rms in their epilogue, fed by the row statistics the o-proj / down-proj GEMMs leave
 * (vsb_gemm_rowscale_bf16) - 6 kernel launches per layer instead of 8.
 * Weight format: the w*_scales fields are NULL for dense weights.  Set, they make the matching w* field hold NF4 codes and
 * themselves the codes' fp32 block scales (layout below), and that projection runs on vsb_gemm_nf4; a table is all dense or
 * all NF4.  NF4 tables need vsb_llama_layers_f16, norm_folded = 0 and tail_rows = 0, and deq_scratch: f16, 2*inter*d elements
 * (the largest weight), which the row counts that take the dequant + tile path use; dense tables leave it unused (NULL). */
typedef struct {
  const void* ln1;
  const void* wqkv;
  const void* wo;
  const void* ln2;
  const void* wgu;
  const void* wdown;
  const void* wqkv_scales;
  const void* wo_scales;
  const void* wgu_scales;
  const void* wdown_scales;
} vsb_llama_layer_t;
int vsb_llama_layers(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int Tn, int past, void* cache, int Bc, int Tmax,
                     int d, int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin, const void* positions,
                     const void* k_start, int tail_rows, const void* q_seg, int seg_lo, int norm_folded, void* scratch,
                     void* deq_scratch, void* stream);
/* f16 twin of vsb_llama_layers: f16 weights, residual stream, cache, RoPE tables and scratch, dispatching to the _f16 kernels */
int vsb_llama_layers_f16(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int Tn, int past, void* cache, int Bc, int Tmax,
                         int d, int H, int inter, float rms_eps, const void* rope_cos, const void* rope_sin, const void* positions,
                         const void* k_start, int tail_rows, const void* q_seg, int seg_lo, int norm_folded, void* scratch,
                         void* deq_scratch, void* stream);

/* Slot decode: one new token for each of B sequences that sit at their OWN cache slot and length, so a decode batch can admit a
 * sequence whenever another one ends (VQAEngine.decode_stream).  slot_i32 / len_i32 / pos_i32: device int32 [B]: row b's cache slot
 * (< Bc, distinct), the rows already cached in it (its new q|k|v row is written at slot*Tmax + len) and its RoPE position.
 * max_len >= every len[b] (< Tmax) sizes the attention launch.  Same per-layer sequence and weight tables (dense or NF4) as
 * vsb_llama_layers with Tn = 1, with the QKV projection written to scratch, placed by vsb_rope_scatter and attended by
 * vsb_attn_decode_slots.  scratch: B*(5d+inter) elements; batch-invariant mode as in vsb_llama_layers.  The three slot-decode
 * entry points take the element type as an argument, dtype = VSB_DTYPE_BF16 or VSB_DTYPE_F16 (f16 and NF4 tables). */
int vsb_llama_layers_slots(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, void* cache, int Bc, int Tmax, int d, int H,
                           int inter, float rms_eps, const void* rope_cos, const void* rope_sin, const void* slot_i32, const void* len_i32,
                           const void* pos_i32, int max_len, int norm_folded, void* scratch, void* deq_scratch, int dtype, void* stream);
/* Row b of qkv [B, 3*H*D] (row stride ldq) to cache row slot_i32[b]*Tmax + len_i32[b] (row stride ldc): q and k rotated at position
 * pos_i32[b] with the arithmetic of vsb_rope_bf16 / vsb_rope_f16, v copied. */
int vsb_rope_scatter(const void* qkv, long long ldq, int B, int H, int D, void* cache, long long ldc, int Tmax, const void* slot_i32,
                     const void* len_i32, const void* pos_i32, const void* cos_table, const void* sin_table, int dtype, void* stream);
/* Decode attention over per-row slots and lengths: row b's query is at q + slot[b]*slot_stride + len[b]*row_stride, and it attends
 * keys / values [0, len[b]] of its slot (k/v + slot[b]*slot_stride + j*row_stride); output o + b*o_rs.  Cluster split-KV as
 * vsb_attn_decode_bf16, with each row's split chosen from its own key count (in batch-invariant mode from nothing else).  In the
 * default mode, with equal lengths and slot[b] = b, it is bit-identical to vsb_attn_decode_bf16 / _f16 (Sq = 1, k_start NULL);
 * in batch-invariant mode it may split differently (vsb_attn_decode_* keeps its batch-size term there).  max_len >= every len[b]. */
int vsb_attn_decode_slots(const void* q, const void* k, const void* v, void* o, long long slot_stride, long long row_stride, long long o_rs,
                          int B, int H, int D, float scale, const void* slot_i32, const void* len_i32, int max_len, int dtype, void* stream);

/* Paged slot decode: the KV cache is a pool of pages of page_rows k|v rows (2d elements per row: k then v), page_rows a power of
 * two >= 16.  page_table_i32 is device int32 [*, pt_ld]; the row of slot s lists its pages, so key row j of slot s sits in page
 * page_table[s*pt_ld + j/page_rows] at row j % page_rows.  Rows of different slots may name the same page (a beam request's
 * shared prompt pages); the caller keeps the pages a step writes private to their slot.
 * vsb_llama_layers_slots_paged: vsb_llama_layers_slots on the pool [n_layers][n_pages][page_rows][2d] (same tables, scratch,
 * dtype and batch-invariant mode), with vsb_rope_scatter_paged / vsb_attn_decode_paged in place of the slot kernels; max_len <
 * pt_ld*page_rows.  Each row's logits are bit-identical to vsb_llama_layers_slots on the same logical keys. */
int vsb_llama_layers_slots_paged(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, void* pool, int n_pages, int page_rows,
                                 const void* page_table_i32, int pt_ld, int d, int H, int inter, float rms_eps, const void* rope_cos,
                                 const void* rope_sin, const void* slot_i32, const void* len_i32, const void* pos_i32, int max_len,
                                 int norm_folded, void* scratch, void* deq_scratch, int dtype, void* stream);
/* vsb_rope_scatter into pages: row b of qkv [B, 3*H*D] (row stride ldq) has q rotated IN PLACE and k rotated at position
 * pos_i32[b]; k|v go to row len_i32[b] of slot slot_i32[b]'s pages (pool + page*page_stride + row*ldc). */
int vsb_rope_scatter_paged(void* qkv, long long ldq, int B, int H, int D, void* pool, long long page_stride, long long ldc, int page_rows,
                           const void* page_table_i32, int pt_ld, const void* slot_i32, const void* len_i32, const void* pos_i32,
                           const void* cos_table, const void* sin_table, int dtype, void* stream);
/* vsb_attn_decode_slots over pages: row b's query at q + b*q_rs, its keys / values [0, len[b]] at k / v + page*page_stride +
 * row*row_stride through slot_i32[b]'s page-table row; output o + b*o_rs.  Same split rule, key chunks and combine as
 * vsb_attn_decode_slots, so the two agree bit for bit on the same logical keys in both modes. */
int vsb_attn_decode_paged(const void* q, long long q_rs, const void* k, const void* v, void* o, long long o_rs, long long page_stride,
                          long long row_stride, int page_rows, const void* page_table_i32, int pt_ld, int B, int H, int D, float scale,
                          const void* slot_i32, const void* len_i32, int max_len, int dtype, void* stream);
/* Chunked prefill over pages: causal attention of R prompt rows in S segments, in one launch.  seg_i32 is device int32 [3][S]
 * (slot, lo, n): segment s holds rows [lo, lo + n) of the request on page-table row slot, its queries are the next n rows of q
 * (row stride ldq; segments back to back, R = sum of n), and query row lo + i attends keys [0, lo + i] of that request.  pool
 * is [pool_rows][2*H*D] k|v rows (k then v) and the layer's pages start at pool row row0: key j sits at pool row row0 +
 * page_table[slot*pt_ld + j/page_rows]*page_rows + j % page_rows.  Output row r at o + r*ldo.  The wgmma flash-attention body
 * of vsb_flash_attn_* with the K/V tiles loaded through the page table, so every row equals that kernel's row on the same
 * logical keys bit for bit; the page rows past a segment's last key may hold anything.  head_dim 64 / 128; page_rows a
 * multiple of 64 (VSB_ERR_ARG otherwise, before any launch). */
int vsb_attn_chunk_paged(const void* q, long long ldq, const void* pool, long long pool_rows, long long row0, void* o, long long ldo,
                         int page_rows, const void* page_table_i32, int pt_ld, const void* seg_i32, int S, int R, int H, int D, float scale,
                         int dtype, void* stream);
/* vsb_llama_layers_slots_paged with R prompt rows appended after the B decode rows (B >= 0, R >= 1): x is [B + R, d] and
 * slot / len / pos int32 [B + R] on the device, chunk row i of a segment (slot, lo, n) having slot, len = pos = lo + i.  The
 * projections and MLP run on all B + R rows, vsb_rope_scatter_paged places every row's k|v, vsb_attn_decode_paged attends the
 * B decode rows (max_len >= their len) and vsb_attn_chunk_paged the R chunk rows (seg_i32 [3][S] as there).  scratch: (B + R)
 * * (5d + inter) elements.  In batch-invariant mode the decode rows equal vsb_llama_layers_slots_paged's and the chunk rows'
 * final hidden states the one-shot vsb_llama_layers prefill's of the whole prompt (Sq >= 64), bit for bit. */
int vsb_llama_layers_chunked_paged(const vsb_llama_layer_t* layers, int n_layers, void* x, int B, int R, void* pool, int n_pages, int page_rows,
                                   const void* page_table_i32, int pt_ld, int d, int H, int inter, float rms_eps, const void* rope_cos,
                                   const void* rope_sin, const void* slot_i32, const void* len_i32, const void* pos_i32, int max_len,
                                   const void* seg_i32, int S, int norm_folded, void* scratch, void* deq_scratch, int dtype, void* stream);
/* vsb_copy_slot_rows_b16 into a paged pool [layers] (layer_stride) of pages: for every pair (src, dst, lo, hi) of the HOST array
 * quads_i32, rows [lo, hi) of every layer are copied to page-table row dst's pages.  src NULL: the source is page-table row src of
 * the pool (a beam fork; the slot rules of vsb_copy_slot_rows_b16 apply).  src set: a contiguous cache, row r of slot s at
 * src + l*src_layer_stride + s*src_slot_stride + r*src_row_stride (a prefilled prompt written into its pages).  row_elems
 * 2-byte elements per row; at most VSB_COPY_ROWS_MAX_PAIRS pairs, slots <= 65536; refusals before any launch.  One launch. */
int vsb_copy_page_rows_b16(void* pool, int layers, long long layer_stride, long long page_stride, int page_rows, long long row_stride,
                           int row_elems, const void* page_table_i32, int pt_ld, int slots, const void* src, long long src_layer_stride,
                           long long src_slot_stride, long long src_row_stride, int src_slots, const int* quads_i32, int npairs,
                           void* stream);
/* Swap whole pages of a paged pool [layers] (layer_stride) of n_pages pages (page_stride; page_elems contiguous 2-byte elements
 * per page) to or from a swap area of PINNED HOST memory [host_slots] (host_slot_stride) [layers] (host_layer_stride): for every
 * pair i of the HOST arrays pages_i32 / slots_i32, to_host != 0 copies page pages_i32[i] of every layer to host slot
 * slots_i32[i], to_host == 0 the other way.  The kernel reads and writes the host area through its mapped device address in
 * 16-byte vectors (pointers and strides must be 16-byte aligned), in stream order with the other launches.  A page or slot out
 * of range, a destination named twice, a null pointer or host memory that is not mapped pinned memory is refused before any
 * launch.  One launch per VSB_SWAP_PAGES_PER_LAUNCH pairs. */
#define VSB_SWAP_PAGES_PER_LAUNCH 384
int vsb_swap_pages_b16(void* pool, int layers, long long layer_stride, int n_pages, long long page_stride, long long page_elems, void* host,
                       int host_slots, long long host_slot_stride, long long host_layer_stride, const int* pages_i32, const int* slots_i32,
                       int n, int to_host, void* stream);

/* NF4 weights: the SEAL VQA LLM's 4-bit mode (the reference's load_4bit: bitsandbytes NF4, double-quantised scales, fp16 compute,
 * LLaVA/llava/model/builder.py:26-43).  Format of W [N, K], K % 64 == 0 (csrc/nf4.cu, oracle/nf4_oracle.py): codes u8 [N, K/2], two
 * 4-bit codes per byte with the first element in the high nibble, one fp32 scale per 64-value block [N, K/64]; a weight is
 * f16(nf4[code] * scale).
 * vsb_nf4_quantize: f16 W -> codes and the first-level fp32 absmax of every block (code = NF4 entry nearest to w * (1/absmax),
 * ties to the lower code).  vsb_nf4_double_quant: absmax [n] -> scales [n] = map[q8] * absmax2 + offset, with offset = *offset (fp32
 * on the device, the mean of absmax), groups of 256, map = the signed 8-bit dynamic map dmap [256] (fp32, sorted). */
int vsb_nf4_quantize(const void* w, int N, int K, void* codes, void* absmax, void* stream);
int vsb_nf4_double_quant(const void* absmax, long long n, const void* offset, const void* dmap, void* scales, void* stream);
/* out [N, K] (row stride ldo) = f16 dequantisation of (codes, scales) */
int vsb_nf4_dequant(const void* codes, const void* scales, int N, int K, void* out, long long ldo, void* stream);
/* vsb_gemm_f16 with W = deq(codes, scales): same arguments, epilogues and semantics.  Small M: weight-streaming kernels that
 * dequantise in registers (vsb_gemm_set_tuning 1 = CUDA-core kernel, M <= 8; 2 = mma.sync kernel, M <= 32); otherwise deq(W) is
 * written to deq_scratch (f16, N*K elements) and vsb_gemm_f16 runs on it (a forced tile width selects this path). */
int vsb_gemm_nf4(const void* A, long long lda, const void* codes, const void* scales, void* C, long long ldc, int M, int N, int K,
                     const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                     long long group_stride, long long group_offset, void* deq_scratch, void* stream);

/* softmax(QK^T*scale [+causal]) V, head_dim 64/128; element (b,s,h,d) at base + b*bs + s*rs + h*D + d.
 * HF CLIP/OWL attention (modeling_clip.py:261-329) and Llama attention (modeling_llama.py:199-221). */
int vsb_flash_attn_bf16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                        long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                        int D, int causal, float scale, void* stream);
/* f16 twin of vsb_flash_attn_bf16 (P goes to P@V as f16) */
int vsb_flash_attn_f16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                       long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                       int D, int causal, float scale, void* stream);
/* Decode attention (Sq <= 4 new rows against a long KV cache; HF Llama attention with past_key_values as driven by
 * generate(use_cache=True), /root/reference/vstar_bench_eval.py:91-103, :127-152): the keys of a head are split over a
 * cluster of 8 CTAs and combined through distributed shared memory.  k_start: optional int32 [B], first valid key of each
 * batch entry (left-padded ragged batches); NULL = 0.  vsb_flash_attn_bf16 routes Sq <= 4 here. */
int vsb_attn_decode_bf16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                         long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                         int D, int causal, float scale, const void* k_start, void* stream);
/* f16 twin of vsb_attn_decode_bf16 */
int vsb_attn_decode_f16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                        long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                        int D, int causal, float scale, const void* k_start, void* stream);
/* Causal attention with a per-row segment mask: the Sq new rows occupy keys Sk-Sq..Sk-1; row r sees keys [0, seg_lo) and
 * [q_seg[b*Sq + r], Sk-Sq+r].  One launch scores every answer option of a question on the question's cached K/V
 * (the reference runs one forward per option on past_key_values, vstar_bench_eval.py:140-152). */
int vsb_flash_attn_seg_bf16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                            long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                            int D, float scale, const void* q_seg_i32, int seg_lo, void* stream);
/* f16 twin of vsb_flash_attn_seg_bf16 */
int vsb_flash_attn_seg_f16(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_rs, long long k_bs,
                           long long k_rs, long long v_bs, long long v_rs, long long o_bs, long long o_rs, int B, int H, int Sq, int Sk,
                           int D, float scale, const void* q_seg_i32, int seg_lo, void* stream);
/* testing hook: 0 = auto (wgmma kernel for Sq >= 64, split-KV decode kernel for Sq <= 4, mma.sync kernel between),
 * 1 = mma.sync, 2 = wgmma, 3 = wgmma with one query warpgroup per CTA only, 4 = decode kernel */
int vsb_attn_set_impl(int impl);
/* SAM two-way transformer attention, head_dim 16/32 (segment_anything/modeling/transformer.py:220-242)
 * and SEAL perceiver-resampler attention, head_dim 96 (LLaVA/llava/model/multimodal_projector/perceiver.py:25-77). */
int vsb_attn_small_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                        int B, int H, int Nq, int Nk, int D, float scale, void* stream);
/* f16 twin of vsb_attn_small_bf16 */
int vsb_attn_small_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                       int B, int H, int Nq, int Nk, int D, float scale, void* stream);

/* OWL-ViT class head epilogue on y = [dense0(x) | logit_shift(x) | logit_scale(x)] (fp32) and box head epilogue
 * (modeling_owlvit.py:1043-1062; owlvit.py:63-100).  quant_bf16 != 0: logits / sigmoid scores / boxes are rounded to bf16
 * VALUES (kept in fp32 storage), which is what the reference's bf16 model hands to the search loop (visual_search.py:145,
 * :223-224, :399-409): thresholds, argmax ties and all_valid_boxes are then decided on the same numbers. */
int vsb_owl_class_post(const void* y, long long ldy, const void* query, long long ldq, int rows_per_crop, long long R, int Q, int quant_bf16,
                       void* logits, void* scores, void* stream);
int vsb_owl_box_post(const void* y, long long ldy, const void* box_bias, int rows_per_crop, long long R, int quant_bf16, void* boxes,
                     void* stream);

/* SAM mask-decoder upscaling helpers (mask_decoder.py:15-27, :78-84, :169-181), channels-last. */
int vsb_upsample2x_nhwc_bf16(const void* x, void* y, int B, int H, int W, int C, void* stream);
int vsb_im2col3x3_nhwc_bf16(const void* x, void* A, int B, int H, int W, int C, void* stream);
int vsb_mask_dot_bf16(const void* up, const void* hyper, void* out, int B, long long P, int C, void* stream);

/* target-cue heatmap: bilinear(align_corners=False) of the fp32 low-res mask to (h,w), optional clamp(min=0),
 * plus (max,min,sum) (VSM.py:534-537; visual_search.py:223-224, :268-275, :420-421). */
int vsb_heatmap_bilinear_f32(const void* low, int LH, int LW, void* out, int h, int w, int do_clamp, void* scratch, void* stats3, void* stream);
/* sums of the min-max-normalised heatmap over integer rectangles [x,y,w,h] (visual_search.py:255-266). */
int vsb_rect_sums_f32(const void* hm, int h, int w, const void* rects_i32, int nrects, const void* stats3, void* out_f64,
                      void* scratch_f64 /* 64*nrects doubles */, void* stream);

/* Crop records (SURVEY.md section 8e): everything the search controller consumes from one crop evaluation as a fixed-size
 * fp32 record rec[row*R ..]: [0] best sigmoid score, [1..4] its cxcywh box, [5] rows P, [6] rows with score > 0.5, [7] best row
 * (-1 = no finite score), [8..10] (max,min,sum) of the clamped target-cue map, [11] number of rectangle sums, [12..75] first 16
 * boxes with score > 0.5 in row order, [76..] rectangle sums.
 * vsb_pack_detections_f32 fills [0..7] and [12..75] for n_crops consecutive records from scores [n,P] / boxes [n,P,4]
 * (argmax with first-index tie-break = torch.argmax; visual_search.py:399-409).
 * vsb_heat_pyramids_f32 fills [8..11] and [76..] for n_jobs crops WITHOUT writing the H x W map: statistics and the sums of the
 * min-max-normalised map over integer rectangles (the crop itself and its quad-tree descendants: get_subpatch_scores over the
 * ancestor chain, visual_search.py:255-275, :453-462) are evaluated from the LH x LW low-res mask with the arithmetic of
 * vsb_heatmap_bilinear_f32 + vsb_rect_sums_f32 (bit-identical).  jobs_i32: 8 ints per job {low_ptr lo, low_ptr hi, h, w, first
 * rect, n_rects, record row, 0}; rects_i32 [total,4] = x,y,w,h relative to the crop; rect_job_i32 [total] = owning job;
 * scratch: 192*n_jobs floats, 64*total_rects doubles. */
int vsb_pack_detections_f32(const void* scores, const void* boxes, int n_crops, int P, void* rec, long long R, void* stream);
int vsb_heat_pyramids_f32(const void* jobs_i32, int n_jobs, const void* rects_i32, const void* rect_job_i32, int total_rects, int LH,
                          int LW, void* rec, long long R, void* scratch_stats_f32, void* scratch_rects_f64, void* stream);

/* Pillow-exact antialiased BICUBIC resize of a uint8 RGB crop resident on the device, in Pillow's two integer passes
 * (libImaging/Resample.c 8bpc path; coefficient tables from vstar_b200/image.py), fused with /255, CLIP mean/std and the
 * bf16 cast.  Replaces the per-crop host preprocessing of visual_search.py:186-194 (PIL crop, expand2square, HF
 * CLIPImageProcessor / OwlViTProcessor resizes, .cuda(), .bfloat16()).  Virtual input = crop (cw x ch at x0,y0 of src)
 * padded bottom/right with bg to in_w x in_h (expand2square, VisualSearch/utils/utils.py:28-39). */
int vsb_resample_h_u8(const void* src, long long row_stride_bytes, int x0, int y0, int cw, int ch, int in_h, int bg0, int bg1, int bg2,
                      const void* coefs_i32, const void* bounds_i32, int ksize, int out_w, void* tmp_u8, void* stream);
int vsb_resample_v_u8(const void* tmp_u8, int out_w, const void* coefs_i32, const void* bounds_i32, int ksize, int out_h, void* out_u8,
                      void* out_bf16_chw, void* out_f32_chw, const float* mean3_host, const float* std3_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VSTAR_B200_H_ */
