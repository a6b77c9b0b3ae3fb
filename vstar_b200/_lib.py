"""ctypes binding of libvstar_b200.so (the C-ABI declared in include/vstar_b200.h).

The product path fails LOUDLY if the library is missing or a call errors: there is no CPU or
PyTorch fallback for any op declared here.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvstar_b200.so")

c_p = ctypes.c_void_p
c_i = ctypes.c_int
c_ll = ctypes.c_longlong
c_f = ctypes.c_float

# name -> argtypes (must match include/vstar_b200.h)
SIGNATURES = {
    "vsb_gemm_bf16": [c_p, c_ll, c_p, c_ll, c_p, c_ll, c_i, c_i, c_i, c_p, c_p, c_ll, c_i, c_i, c_i, c_ll, c_ll, c_p],
    "vsb_set_batch_invariant": [c_i],
    "vsb_gemm_profile_begin": [],
    "vsb_gemm_profile_end": [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(c_ll)],
    "vsb_gemm_set_tuning": [c_i, c_i],
    "vsb_gemm_set_group_m": [c_i],
    "vsb_gemm_set_l2_hints": [c_i],
    "vsb_layernorm_bf16": [c_p, c_ll, c_p, c_p, c_p, c_ll, c_i, c_i, c_f, c_i, c_p],
    "vsb_rmsnorm_bf16": [c_p, c_ll, c_p, c_p, c_ll, c_i, c_i, c_f, c_p],
    "vsb_rope_bf16": [c_p, c_ll, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_p, c_ll, c_ll, c_p],
    "vsb_embed_splice_bf16": [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, c_p],
    "vsb_gather_rows_bf16": [c_p, c_p, c_ll, c_p, c_ll, c_i, c_i, c_ll, c_p],
    "vsb_patchify_bf16": [c_p, c_p, c_i, c_i, c_i, c_i, c_p],
    "vsb_vit_add_pos_bf16": [c_p, c_p, c_p, c_i, c_i, c_i, c_p],
    "vsb_owl_merge_bf16": [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_f, c_p],
    "vsb_add_rows_bf16": [c_p, c_p, c_p, c_ll, c_i, c_ll, c_p],
    "vsb_cast_f32_bf16": [c_p, c_p, c_ll, c_p],
    "vsb_nll_rows_f32": [c_p, c_ll, c_i, c_i, c_p, c_p, c_p],
    "vsb_argmax_rows_f32": [c_p, c_ll, c_i, c_i, c_p, c_p, c_p],
    "vsb_sample_rows_f32": [c_p, c_ll, c_i, c_i, c_f, c_i, c_f, c_i, c_p, c_i, c_p, c_p],
    "vsb_sample_rows_var_f32": [c_p, c_ll, c_i, c_i, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_p],
    "vsb_copy2d_b16": [c_p, c_ll, c_p, c_ll, c_ll, c_i, c_p],
    "vsb_beam_candidates_f32": [c_p, c_ll, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_p, c_p, c_p, c_p],
    "vsb_copy_cache_rows_b16": [c_p, c_i, c_ll, c_i, c_ll, c_ll, c_i, c_p, c_i, c_i, c_i, c_p],
    "vsb_copy_slot_rows_b16": [c_p, c_i, c_ll, c_i, c_ll, c_ll, c_i, c_p, c_i, c_p],
    "vsb_llama_layers": [c_p, c_i, c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_p, c_p, c_i, c_p, c_i, c_i, c_p, c_p,
                         c_p],
    "vsb_gemm_rowscale_bf16": [c_p, c_ll, c_p, c_ll, c_p, c_ll, c_i, c_i, c_i, c_p, c_p, c_ll, c_i, c_i, c_ll, c_ll, c_p, c_i, c_f, c_p, c_ll, c_p],
    "vsb_rowsq_bf16": [c_p, c_ll, c_p, c_i, c_i, c_p],
    "vsb_gemm_qkv_rope_bf16": [c_p, c_ll, c_p, c_ll, c_p, c_ll, c_i, c_i, c_i, c_i, c_ll, c_ll, c_p, c_i, c_f, c_ll, c_p, c_p, c_p, c_i, c_i, c_i, c_p],
    "vsb_llama_set_fuse_rope": [c_i],
    "vsb_flash_attn_seg_bf16": [c_p, c_p, c_p, c_p, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_i, c_i, c_i, c_i, c_i, c_f, c_p, c_i, c_p],
    "vsb_attn_decode_bf16": [c_p, c_p, c_p, c_p, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_i, c_i, c_i, c_i, c_i, c_i, c_f, c_p, c_p],
    "vsb_flash_attn_bf16": [c_p, c_p, c_p, c_p, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_ll, c_i, c_i, c_i, c_i, c_i, c_i, c_f, c_p],
    "vsb_attn_set_impl": [c_i],
    "vsb_attn_small_bf16": [c_p, c_ll, c_p, c_ll, c_p, c_ll, c_p, c_ll, c_i, c_i, c_i, c_i, c_i, c_f, c_p],
    "vsb_owl_class_post": [c_p, c_ll, c_p, c_ll, c_i, c_ll, c_i, c_i, c_p, c_p, c_p],
    "vsb_owl_box_post": [c_p, c_ll, c_p, c_i, c_ll, c_i, c_p, c_p],
    "vsb_pack_detections_f32": [c_p, c_p, c_i, c_i, c_p, c_ll, c_p],
    "vsb_heat_pyramids_f32": [c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_p, c_ll, c_p, c_p, c_p],
    "vsb_upsample2x_nhwc_bf16": [c_p, c_p, c_i, c_i, c_i, c_i, c_p],
    "vsb_im2col3x3_nhwc_bf16": [c_p, c_p, c_i, c_i, c_i, c_i, c_p],
    "vsb_mask_dot_bf16": [c_p, c_p, c_p, c_i, c_ll, c_i, c_p],
    "vsb_heatmap_bilinear_f32": [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_p, c_p],
    "vsb_rect_sums_f32": [c_p, c_i, c_i, c_p, c_i, c_p, c_p, c_p, c_p],
    "vsb_resample_h_u8": [c_p, c_ll, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_i, c_p, c_p],
    "vsb_resample_v_u8": [c_p, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p, ctypes.POINTER(c_f), ctypes.POINTER(c_f), c_p],
}

# f16 twins (same argument types as their _bf16 siblings): the SEAL VQA LLM in fp16
for _name in ("vsb_gemm", "vsb_gemm_rowscale", "vsb_gemm_qkv_rope", "vsb_rowsq", "vsb_layernorm", "vsb_rmsnorm", "vsb_rope", "vsb_add_rows",
              "vsb_vit_add_pos", "vsb_cast_f32", "vsb_flash_attn", "vsb_attn_decode", "vsb_flash_attn_seg", "vsb_attn_small"):
    SIGNATURES[_name + "_f16"] = SIGNATURES[_name + "_bf16"]
SIGNATURES["vsb_llama_layers_f16"] = SIGNATURES["vsb_llama_layers"]

# NF4 weights (the SEAL VQA LLM's 4-bit mode)
SIGNATURES.update({
    "vsb_nf4_quantize": [c_p, c_i, c_i, c_p, c_p, c_p],
    "vsb_nf4_double_quant": [c_p, c_ll, c_p, c_p, c_p, c_p],
    "vsb_nf4_dequant": [c_p, c_p, c_i, c_i, c_p, c_ll, c_p],
    "vsb_gemm_nf4": [c_p, c_ll, c_p, c_p, c_p, c_ll, c_i, c_i, c_i, c_p, c_p, c_ll, c_i, c_i, c_i, c_ll, c_ll, c_p, c_p],
})

# slot decode (VQAEngine.decode_stream): every row at its own cache slot and length; the element type is an argument
SIGNATURES.update({
    "vsb_llama_layers_slots": [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i, c_p],
    "vsb_rope_scatter": [c_p, c_ll, c_i, c_i, c_i, c_p, c_ll, c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_p],
    "vsb_attn_decode_slots": [c_p, c_p, c_p, c_p, c_ll, c_ll, c_ll, c_i, c_i, c_i, c_f, c_p, c_p, c_i, c_i, c_p],
})

# paged slot decode (DecodeStream(kv_pages=N)): k|v rows in pages found through a device page table
SIGNATURES.update({
    "vsb_llama_layers_slots_paged": [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p,
                                     c_p, c_i, c_p],
    "vsb_rope_scatter_paged": [c_p, c_ll, c_i, c_i, c_i, c_p, c_ll, c_ll, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_p],
    "vsb_attn_decode_paged": [c_p, c_ll, c_p, c_p, c_p, c_ll, c_ll, c_ll, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_i, c_i, c_p],
    "vsb_copy_page_rows_b16": [c_p, c_i, c_ll, c_ll, c_i, c_ll, c_i, c_p, c_i, c_i, c_p, c_ll, c_ll, c_ll, c_i, c_p, c_i, c_p],
    "vsb_swap_pages_b16": [c_p, c_i, c_ll, c_i, c_ll, c_ll, c_p, c_i, c_ll, c_ll, c_p, c_p, c_i, c_i, c_p],
})

# chunked prefill on the paged stream (DecodeStream(kv_pages=N, prefill_chunk=C)): prompt rows ride along with the decode rows
SIGNATURES.update({
    "vsb_attn_chunk_paged": [c_p, c_ll, c_p, c_ll, c_ll, c_p, c_ll, c_i, c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_i, c_p],
    "vsb_llama_layers_chunked_paged": [c_p, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_p, c_p, c_p, c_i,
                                       c_p, c_i, c_i, c_p, c_p, c_i, c_p],
})


class LlamaLayer(ctypes.Structure):
    """vsb_llama_layer_t"""
    _fields_ = [("ln1", c_p), ("wqkv", c_p), ("wo", c_p), ("ln2", c_p), ("wgu", c_p), ("wdown", c_p),
                ("wqkv_scales", c_p), ("wo_scales", c_p), ("wgu_scales", c_p), ("wdown_scales", c_p)]


_lib = None


class VsbError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VsbError(
            f"{LIB_PATH} not found: build it with `python -m vstar_b200.build` "
            "(there is NO CPU / PyTorch fallback for the vstar_b200 kernels)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.vsb_last_error.restype = ctypes.c_char_p
    lib.vsb_last_error.argtypes = []
    lib.vsb_version.restype = c_i
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the symbol is missing
        fn.argtypes = args
        fn.restype = c_i
    _lib = lib
    return lib


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise VsbError(f"{name} failed ({rc}): {lib.vsb_last_error().decode()}")
    return rc


# launch counter (bench.py reports gpu_launches from it)
launches = 0
