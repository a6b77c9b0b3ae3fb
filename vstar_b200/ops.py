"""Tensor-level wrappers over the C-ABI (torch is only the owner of device memory and streams here).

Every function launches hand-written sm_90a kernels from libvstar_b200.so on the current torch CUDA
stream.  No function has a PyTorch fallback: on a box without the built library, or on CPU tensors,
they raise.

The ops of the SEAL VQA LLM's path dispatch on the operand dtype: bf16 tensors run the _bf16 kernels, fp16 tensors their _f16
twins.  Operands of one call must share that dtype (VsbError otherwise); the VSM-only ops are bf16-only.
"""
import torch

from . import _lib
from ._lib import call

EPI_NONE, EPI_QUICK_GELU, EPI_GELU, EPI_RELU, EPI_SWIGLU = 0, 1, 2, 3, 4
BF16 = torch.bfloat16
F16 = torch.float16
_SUFFIX = {BF16: "bf16", F16: "f16"}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _chk(t, dtype=None):
    if not t.is_cuda:
        raise _lib.VsbError("vstar_b200 ops need CUDA tensors (no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise _lib.VsbError(f"expected {dtype}, got {t.dtype}")
    return t


def _sfx(*ts):
    """kernel variant ("bf16" / "f16") for the dtype shared by all given tensors (None entries are skipped)"""
    dt = None
    for t in ts:
        if t is None:
            continue
        _chk(t)
        if dt is None:
            dt = t.dtype
        elif t.dtype != dt:
            raise _lib.VsbError(f"mixed operand dtypes {dt} and {t.dtype} (one call runs on bf16 or on fp16 operands)")
    if dt not in _SUFFIX:
        raise _lib.VsbError(f"unsupported dtype {dt}: the kernels take bf16 or fp16")
    return _SUFFIX[dt]


def _rows2d(t):
    """(ptr, rows, cols, ld) of a 2-D row-major view with unit inner stride."""
    assert t.dim() == 2 and t.stride(1) == 1, (t.shape, t.stride())
    return t.data_ptr(), t.shape[0], t.shape[1], t.stride(0)


class batch_invariant:
    """with ops.batch_invariant(): kernels are chosen independently of the row count of a call (see vsb_set_batch_invariant)"""
    depth = 0

    def __enter__(self):
        if batch_invariant.depth == 0:
            call("vsb_set_batch_invariant", 1)
        batch_invariant.depth += 1

    def __exit__(self, *a):
        batch_invariant.depth -= 1
        if batch_invariant.depth == 0:
            call("vsb_set_batch_invariant", 0)


# optional per-launch profiling of the dominant kernel (bench.py roofline): CUDA events around every GEMM launch
profiling = False


def profile_begin():
    """CUDA events around every vsb_gemm_bf16 launch from here on (recorded inside the library, so launches issued by the native
    layer runner are covered too)"""
    global profiling
    profiling = True
    call("vsb_gemm_profile_begin")


def profile_end():
    """-> (total algorithmic flops, total ms, launches) over the GEMM launches since profile_begin()"""
    import ctypes
    global profiling
    f, t, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
    call("vsb_gemm_profile_end", ctypes.byref(f), ctypes.byref(t), ctypes.byref(n))
    profiling = False
    return f.value, t.value, n.value


NF4_LINEARS = ("wqkv", "wo", "wgu", "wdown")


class NF4Weight:
    """A weight W [N, K] in NF4 (the SEAL VQA LLM's 4-bit mode, see include/vstar_b200.h): codes uint8 [N, K/2] (first element of
    a pair in the high nibble) and fp32 scales [N, K/64], one per 64-value block.  W dequantises to f16(nf4[code] * scale)."""

    def __init__(self, codes, scales, N, K):
        assert codes.dtype == torch.uint8 and codes.shape == (N, K // 2) and codes.is_contiguous()
        assert scales.dtype == torch.float32 and scales.shape == (N, K // 64) and scales.is_contiguous()
        self.codes, self.scales, self.N, self.K = codes, scales, N, K

    @property
    def shape(self):
        return (self.N, self.K)

    @property
    def nbytes(self):
        return self.codes.numel() + 4 * self.scales.numel()

    @staticmethod
    def cat_rows(ws):
        """rows of several NF4 weights of the same K stacked (wqkv = q | k | v)"""
        assert len({w.K for w in ws}) == 1
        return NF4Weight(torch.cat([w.codes for w in ws], 0), torch.cat([w.scales for w in ws], 0), sum(w.N for w in ws), ws[0].K)

    @staticmethod
    def interleave_rows(a, b):
        """row 2j = a_j, row 2j+1 = b_j (wgu: gate / up)"""
        assert a.shape == b.shape
        return NF4Weight(torch.stack([a.codes, b.codes], 1).reshape(2 * a.N, -1).contiguous(),
                         torch.stack([a.scales, b.scales], 1).reshape(2 * a.N, -1).contiguous(), 2 * a.N, a.K)


def weight_nbytes(w):
    """device bytes of a dense or NF4 weight"""
    return w.nbytes if isinstance(w, NF4Weight) else w.numel() * w.element_size()


def nf4_dynamic_map(device):
    """bitsandbytes' create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8): 256 sorted fp32 values"""
    data = []
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** i + 1)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-6 + i)) * means).tolist()
        data += (-(10 ** (-6 + i)) * means).tolist()
    data += [0.0, 1.0]
    data.sort()
    return torch.tensor(data, dtype=torch.float32).to(device)


_DMAP = {}


def nf4_quantize(w):
    """fp16 [N, K] CUDA tensor (K % 64 == 0) -> NF4Weight, with bitsandbytes' double quant of the block scales (offset = mean of
    the block absmax, taken on the device)"""
    _chk(w, F16)
    assert w.dim() == 2 and w.is_contiguous()
    N, K = w.shape
    if K % 64:
        raise _lib.VsbError(f"NF4 needs K % 64 == 0 (64-value blocks inside one row), got K = {K}")
    codes = torch.empty((N, K // 2), dtype=torch.uint8, device=w.device)
    absmax = torch.empty((N, K // 64), dtype=torch.float32, device=w.device)
    _lib.launches += 2
    call("vsb_nf4_quantize", w.data_ptr(), N, K, codes.data_ptr(), absmax.data_ptr(), _stream())
    offset = absmax.mean()
    dmap = _DMAP.get(w.device)
    if dmap is None:
        dmap = _DMAP[w.device] = nf4_dynamic_map(w.device)
    scales = torch.empty_like(absmax)
    call("vsb_nf4_double_quant", absmax.data_ptr(), absmax.numel(), offset.data_ptr(), dmap.data_ptr(), scales.data_ptr(), _stream())
    return NF4Weight(codes, scales, N, K)


def nf4_dequant(w, out=None):
    """NF4Weight -> fp16 [N, K] (into `out`, a view with unit inner stride, if given)"""
    if out is None:
        out = torch.empty((w.N, w.K), dtype=F16, device=w.codes.device)
    _chk(out, F16)
    assert out.shape == (w.N, w.K) and out.stride(1) == 1
    _lib.launches += 1
    call("vsb_nf4_dequant", w.codes.data_ptr(), w.scales.data_ptr(), w.N, w.K, out.data_ptr(), out.stride(0), _stream())
    return out


def _layer_nf4(L):
    return isinstance(L["wqkv"], NF4Weight)


def llama_layer_table(layers):
    """layers: list of dicts with ln1, wqkv, wo, ln2, wgu, wdown tensors (kept alive by the caller), all bf16 or all fp16
    -> vsb_llama_layer_t ctypes array.  NF4 layers (wqkv, wo, wgu, wdown NF4Weight, fp16 ln1 / ln2) fill the codes into the
    weight fields and their scales into the *_scales fields; a table cannot mix NF4 and dense layers."""
    nf4 = _layer_nf4(layers[0])
    if any(isinstance(L[k], NF4Weight) != nf4 for L in layers for k in NF4_LINEARS):
        raise _lib.VsbError("a layer table cannot mix NF4 and fp16 / bf16 projections")
    arr = (_lib.LlamaLayer * len(layers))()
    dtypes = set()
    for i, L in enumerate(layers):
        for k in ("ln1", "wqkv", "wo", "ln2", "wgu", "wdown"):
            t = L[k]
            if isinstance(t, NF4Weight):
                setattr(arr[i], k + "_scales", t.scales.data_ptr())
                t = t.codes
            else:
                dtypes.add(t.dtype)
                assert t.dtype in _SUFFIX and t.is_contiguous() and t.is_cuda, k
            setattr(arr[i], k, t.data_ptr())
    if len(dtypes) > 1:
        raise _lib.VsbError(f"mixed layer weight dtypes {sorted(map(str, dtypes))}")
    if nf4 and dtypes != {F16}:
        raise _lib.VsbError(f"NF4 layers take fp16 ln1 / ln2, got {dtypes.pop()}")
    return arr


def llama_layers(table, n_layers, x, B, Tn, past, cache, Bc, Tmax, d, H, inter, eps, rope_cos, rope_sin, scratch, positions=None,
                 k_start=None, cache_row_offset=0, tail_rows=0, q_seg=None, seg_lo=0, norm_folded=False, deq_scratch=None):
    """whole decoder stack in ONE native call (csrc/llama_layers.cu): in place on x [B*Tn, d].
    cache_row_offset shifts the cache origin by that many [3d] rows (a sequence placed at batch slot b, first row s:
    b*Tmax + s) so a single sequence can be prefilled anywhere in a shared cache; positions / k_start: ragged decode;
    tail_rows > 0: only the last tail_rows rows of every sequence are valid on return (the last layer skips the others);
    q_seg int32 [B*Tn] + seg_lo: the new rows are several continuations of the cached prefix [0, seg_lo) appended back to back;
    row r attends the prefix and its own continuation from key q_seg[r] on;
    norm_folded: ln1 / ln2 are already multiplied into wqkv / wgu (fused RMSNorm path, see vsb_llama_layers).
    x, cache, scratch, the RoPE tables and the table's weights are all bf16 or all fp16 (vsb_llama_layers_f16).
    An NF4 table (fp16 only, norms not folded, tail_rows 0) needs deq_scratch, fp16 with 2 * inter * d elements."""
    sfx = _sfx(x, cache, scratch, rope_cos, rope_sin)
    fn = "vsb_llama_layers" if sfx == "bf16" else "vsb_llama_layers_f16"
    assert x.is_contiguous() and cache.is_contiguous() and x.shape == (B * Tn, d)
    assert scratch.numel() >= B * Tn * (2 * d + inter)
    for t in (positions, k_start, q_seg):
        assert t is None or (t.dtype == torch.int32 and t.is_contiguous() and t.is_cuda)
    assert q_seg is None or (q_seg.numel() == B * Tn and positions is not None)
    assert positions is None or positions.numel() == B * Tn
    assert k_start is None or k_start.numel() == B
    if table[0].wqkv_scales:                    # NF4 table
        if sfx != "f16" or norm_folded or tail_rows:
            raise _lib.VsbError("NF4 layers run in fp16 with unfolded norms and tail_rows = 0")
        _chk(deq_scratch, F16)
        assert deq_scratch.is_contiguous() and deq_scratch.numel() >= 2 * inter * d
        _lib.launches += 9 * n_layers
    else:
        _lib.launches += (6 if (norm_folded and k_start is None and (B * Tn > 16 or batch_invariant.depth > 0)) else 8) * n_layers + \
            (2 if (tail_rows > 0 and 2 * tail_rows <= Tn and k_start is None) else 0)
    call(fn, table, n_layers, x.data_ptr(), B, Tn, past, cache.data_ptr() + cache_row_offset * 3 * d * 2, Bc, Tmax, d, H,
         inter, float(eps), rope_cos.data_ptr(), rope_sin.data_ptr(), _p(positions), _p(k_start), int(tail_rows), _p(q_seg), int(seg_lo),
         1 if norm_folded else 0, scratch.data_ptr(), _p(deq_scratch), _stream())
    return x


_DTYPE = {"bf16": 0, "f16": 1}                 # VSB_DTYPE_BF16 / VSB_DTYPE_F16


def _i32_rows(*ts, n):
    for t in ts:
        assert t.dtype == torch.int32 and t.is_contiguous() and t.is_cuda and t.numel() == n


def llama_layers_slots(table, n_layers, x, cache, eps, rope_cos, rope_sin, scratch, slot, length, pos, max_len, H, inter,
                       norm_folded=False, deq_scratch=None):
    """one decode step of B sequences that each sit at their own slot and length of cache [n_layers, Bc, Tmax, 3d]
    (vsb_llama_layers_slots): in place on x [B, d]; slot / length / pos int32 [B] on the device (row b's new q|k|v goes to
    cache row slot[b]*Tmax + length[b] at RoPE position pos[b], and it attends rows [0, length[b]]); max_len >= max(length).
    scratch: B * (5d + inter) elements; NF4 tables as in llama_layers."""
    sfx = _sfx(x, cache, scratch, rope_cos, rope_sin)
    B, d = x.shape
    L, Bc, Tmax, W = cache.shape
    assert x.is_contiguous() and cache.is_contiguous() and W == 3 * d and L >= n_layers
    assert scratch.numel() >= B * (5 * d + inter)
    _i32_rows(slot, length, pos, n=B)
    if table[0].wqkv_scales:
        if sfx != "f16" or norm_folded:
            raise _lib.VsbError("NF4 layers run in fp16 with unfolded norms")
        _chk(deq_scratch, F16)
        assert deq_scratch.is_contiguous() and deq_scratch.numel() >= 2 * inter * d
    _lib.launches += 8 * n_layers
    call("vsb_llama_layers_slots", table, n_layers, x.data_ptr(), B, cache.data_ptr(), Bc, Tmax, d, H, inter, float(eps), rope_cos.data_ptr(),
         rope_sin.data_ptr(), slot.data_ptr(), length.data_ptr(), pos.data_ptr(), int(max_len), 1 if norm_folded else 0, scratch.data_ptr(),
         _p(deq_scratch), _DTYPE[sfx], _stream())
    return x


def _pool_shape(pool, page_table):
    """pool [n_layers, n_pages, P, 2d] or one layer's [n_pages, P, 2d], page_table int32 [rows, pages_per_row] -> (P, pages_per_row)"""
    assert pool.is_contiguous() and pool.dim() in (3, 4)
    P = pool.shape[-2]
    if P < 16 or P & (P - 1):
        raise _lib.VsbError(f"page rows {P} is not a power of two >= 16")
    _chk(page_table, torch.int32)
    assert page_table.dim() == 2 and page_table.is_contiguous()
    return P, page_table.shape[1]


def llama_layers_slots_paged(table, n_layers, x, pool, page_table, eps, rope_cos, rope_sin, scratch, slot, length, pos, max_len, H, inter,
                             norm_folded=False, deq_scratch=None):
    """llama_layers_slots on a paged KV pool [n_layers, n_pages, P, 2d] of k|v rows (vsb_llama_layers_slots_paged): row b's
    keys are rows [0, length[b]] of the pages page_table[slot[b]] lists (page_table int32 [rows, pages_per_row] on the device),
    its new k|v go to row length[b]; max_len >= max(length) and < pages_per_row * P.  scratch, NF4 tables as llama_layers_slots."""
    sfx = _sfx(x, pool, scratch, rope_cos, rope_sin)
    B, d = x.shape
    L, n_pages, P, W = pool.shape
    P, ppr = _pool_shape(pool, page_table)
    assert x.is_contiguous() and W == 2 * d and L >= n_layers
    assert scratch.numel() >= B * (5 * d + inter)
    _i32_rows(slot, length, pos, n=B)
    if table[0].wqkv_scales:
        if sfx != "f16" or norm_folded:
            raise _lib.VsbError("NF4 layers run in fp16 with unfolded norms")
        _chk(deq_scratch, F16)
        assert deq_scratch.is_contiguous() and deq_scratch.numel() >= 2 * inter * d
    _lib.launches += 8 * n_layers
    call("vsb_llama_layers_slots_paged", table, n_layers, x.data_ptr(), B, pool.data_ptr(), n_pages, P, page_table.data_ptr(), ppr, d, H, inter,
         float(eps), rope_cos.data_ptr(), rope_sin.data_ptr(), slot.data_ptr(), length.data_ptr(), pos.data_ptr(), int(max_len),
         1 if norm_folded else 0, scratch.data_ptr(), _p(deq_scratch), _DTYPE[sfx], _stream())
    return x


def llama_layers_chunked_paged(table, n_layers, x, pool, page_table, eps, rope_cos, rope_sin, scratch, slot, length, pos, max_len, seg,
                               chunk_rows, H, inter, norm_folded=False, deq_scratch=None):
    """llama_layers_slots_paged on B decode rows followed by R = chunk_rows prompt rows (vsb_llama_layers_chunked_paged): x [B + R, d]
    in place; slot / length / pos int32 [B + R] on the device (chunk row i of segment (slot, lo, n) has length = pos = lo + i); seg
    int32 [3, S] on the device (slot, lo, n per segment; R = the sum of n); max_len >= the decode rows' lengths.
    scratch: (B + R) * (5d + inter) elements; NF4 tables as in llama_layers_slots."""
    sfx = _sfx(x, pool, scratch, rope_cos, rope_sin)
    rows, d = x.shape
    L, n_pages, P, W = pool.shape
    P, ppr = _pool_shape(pool, page_table)
    assert x.is_contiguous() and W == 2 * d and L >= n_layers
    assert scratch.numel() >= rows * (5 * d + inter)
    _i32_rows(slot, length, pos, n=rows)
    _chk(seg, torch.int32)
    assert seg.dim() == 2 and seg.shape[0] == 3 and seg.is_contiguous()
    S, R = seg.shape[1], int(chunk_rows)
    assert 1 <= R <= rows
    if table[0].wqkv_scales:
        if sfx != "f16" or norm_folded:
            raise _lib.VsbError("NF4 layers run in fp16 with unfolded norms")
        _chk(deq_scratch, F16)
        assert deq_scratch.is_contiguous() and deq_scratch.numel() >= 2 * inter * d
    _lib.launches += 8 * n_layers
    call("vsb_llama_layers_chunked_paged", table, n_layers, x.data_ptr(), rows - R, R, pool.data_ptr(), n_pages, P, page_table.data_ptr(), ppr,
         d, H, inter, float(eps), rope_cos.data_ptr(), rope_sin.data_ptr(), slot.data_ptr(), length.data_ptr(), pos.data_ptr(), int(max_len),
         seg.data_ptr(), S, 1 if norm_folded else 0, scratch.data_ptr(), _p(deq_scratch), _DTYPE[sfx], _stream())
    return x


def attn_chunk_paged(q, pool, page_table, out, H, D, scale, seg, layer=0):
    """causal attention of prompt-chunk rows over a paged pool [n_layers, n_pages, P, 2*H*D] (or one layer's [n_pages, P, 2*H*D]) of
    k|v rows, P a multiple of 64 (vsb_attn_chunk_paged): seg int32 [3, S] on the device lists (slot, lo, n) per segment; the
    segments' query rows are q's rows back to back (q [R, >= H*D], unit inner stride), and row lo + i of segment s attends keys
    [0, lo + i] of the pages page_table[slot] lists in layer `layer` -> out [R, H*D]"""
    sfx = _sfx(q, pool, out)
    pq, R, _, ldq = _rows2d(q)
    P, ppr = _pool_shape(pool, page_table)
    assert pool.shape[-1] == 2 * H * D and out.stride(1) == 1 and out.shape[0] == R
    _chk(seg, torch.int32)
    assert seg.dim() == 2 and seg.shape[0] == 3 and seg.is_contiguous()
    pool_rows = pool.numel() // pool.shape[-1]
    row0 = layer * (pool.shape[-3] * P)
    _lib.launches += 1
    call("vsb_attn_chunk_paged", pq, ldq, pool.data_ptr(), pool_rows, row0, out.data_ptr(), out.stride(0), P, page_table.data_ptr(), ppr,
         seg.data_ptr(), seg.shape[1], R, H, D, float(scale), _DTYPE[sfx], _stream())
    return out


def rope_scatter_paged(qkv, pool, page_table, H, D, cos_t, sin_t, slot, length, pos):
    """rope_scatter into one layer's pages [n_pages, P, 2*H*D] (vsb_rope_scatter_paged): row b of qkv [B, 3*H*D] has q rotated in
    place, its rotated k and its v go to row length[b] of the pages page_table[slot[b]] lists"""
    sfx = _sfx(qkv, pool, cos_t, sin_t)
    p, B, cols, ld = _rows2d(qkv)
    P, ppr = _pool_shape(pool, page_table)
    assert cols == 3 * H * D and pool.dim() == 3 and pool.shape[2] == 2 * H * D
    _i32_rows(slot, length, pos, n=B)
    _lib.launches += 1
    call("vsb_rope_scatter_paged", p, ld, B, H, D, pool.data_ptr(), pool.stride(0), pool.stride(1), P, page_table.data_ptr(), ppr,
         slot.data_ptr(), length.data_ptr(), pos.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), _DTYPE[sfx], _stream())
    return pool


def attn_decode_paged(q, pool, page_table, out, H, D, scale, slot, length, max_len=None):
    """attn_decode_slots over one layer's pages [n_pages, P, 2*H*D] (vsb_attn_decode_paged): row b's query is q[b, :H*D] and it
    attends rows [0, length[b]] of the pages page_table[slot[b]] lists -> out [B, H*D]"""
    sfx = _sfx(q, pool, out)
    pq, B, _, ldq = _rows2d(q)
    P, ppr = _pool_shape(pool, page_table)
    assert pool.dim() == 3 and pool.shape[2] == 2 * H * D and out.stride(1) == 1 and out.shape[0] == B
    _i32_rows(slot, length, n=B)
    if max_len is None:
        max_len = int(length.max())
    base = pool.data_ptr()
    _lib.launches += 1
    call("vsb_attn_decode_paged", pq, ldq, base, base + 2 * H * D, out.data_ptr(), out.stride(0), pool.stride(0), pool.stride(1), P,
         page_table.data_ptr(), ppr, B, H, D, float(scale), slot.data_ptr(), length.data_ptr(), int(max_len), _DTYPE[sfx], _stream())
    return out


def copy_page_rows(pool, page_table, quads, src=None):
    """rows [lo, hi) of every layer into page-table row d's pages of pool [L, n_pages, P, W] for every (s, d, lo, hi) in the host
    list `quads`, in one vsb_copy_page_rows_b16 launch (at most COPY_ROWS_MAX_PAIRS pairs).  src None: from page-table row s of
    the pool (the rules of copy_slot_rows); src a [L, S, T, >= W] view with unit inner stride (e.g. the k|v columns of a fused
    q|k|v cache): from its slot s."""
    import ctypes
    _chk(pool)
    assert pool.dim() == 4 and pool.element_size() == 2
    P, ppr = _pool_shape(pool, page_table)
    L, _, _, W = pool.shape
    if src is None:
        sp, sls, sss, srs, ns = None, 0, 0, 0, 0
    else:
        _chk(src, pool.dtype)
        assert src.dim() == 4 and src.shape[0] == L and src.shape[3] == W and src.stride(3) == 1
        sp, sls, sss, srs, ns = src.data_ptr(), src.stride(0), src.stride(1), src.stride(2), src.shape[1]
    arr = (ctypes.c_int * (4 * max(1, len(quads))))(*[int(v) for q in quads for v in q])
    _lib.launches += 1
    call("vsb_copy_page_rows_b16", pool.data_ptr(), L, pool.stride(0), pool.stride(1), P, pool.stride(2), W, page_table.data_ptr(), ppr,
         page_table.shape[0], sp, sls, sss, srs, ns, arr, len(quads), _stream())
    return pool


def swap_pages(pool, host, pairs, to_host):
    """whole pages of every layer between pool [L, n_pages, P, W] and the pinned host swap area host [M, L, P, W] of the same
    2-byte dtype (vsb_swap_pages_b16): for every (page, slot) in the host list `pairs`, page -> host slot when to_host, else
    host slot -> page.  Runs on the current stream with no host synchronisation; one launch per SWAP_PAGES_PER_LAUNCH pairs."""
    import ctypes
    _chk(pool)
    if host.is_cuda or not host.is_pinned() or host.dtype != pool.dtype:
        raise _lib.VsbError("the swap area must be pinned host memory of the pool's dtype")
    assert pool.dim() == 4 and pool.element_size() == 2 and pool.is_contiguous() and host.is_contiguous()
    assert host.dim() == 4 and tuple(host.shape[1:]) == (pool.shape[0],) + tuple(pool.shape[2:])
    n = len(pairs)
    pages = (ctypes.c_int * max(1, n))(*[int(p) for p, _ in pairs])
    slots = (ctypes.c_int * max(1, n))(*[int(s) for _, s in pairs])
    _lib.launches += -(-n // SWAP_PAGES_PER_LAUNCH)
    call("vsb_swap_pages_b16", pool.data_ptr(), pool.shape[0], pool.stride(0), pool.shape[1], pool.stride(1), pool.shape[2] * pool.shape[3],
         host.data_ptr(), host.shape[0], host.stride(0), host.stride(1), pages, slots, n, 1 if to_host else 0, _stream())
    return pool


def rope_scatter(qkv, cache, H, D, cos_t, sin_t, slot, length, pos):
    """row b of qkv [B, 3*H*D] -> cache row slot[b]*Tmax + length[b] of cache [Bc, Tmax, 3*H*D] (one layer), q and k rotated at
    position pos[b] like rope_, v copied (vsb_rope_scatter)"""
    sfx = _sfx(qkv, cache, cos_t, sin_t)
    p, B, cols, ld = _rows2d(qkv)
    assert cols == 3 * H * D and cache.dim() == 3 and cache.shape[2] == cols and cache.is_contiguous()
    _i32_rows(slot, length, pos, n=B)
    _lib.launches += 1
    call("vsb_rope_scatter", p, ld, B, H, D, cache.data_ptr(), cache.stride(1), cache.shape[1], slot.data_ptr(), length.data_ptr(),
         pos.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), _DTYPE[sfx], _stream())
    return cache


def attn_decode_slots(cache, out, H, D, scale, slot, length, max_len=None):
    """decode attention over per-row slots and lengths (vsb_attn_decode_slots) on one layer's fused cache [Bc, Tmax, 3*H*D]:
    row b's query is cache[slot[b], length[b], :H*D] and it attends rows [0, length[b]] of its slot -> out [B, H*D].
    max_len: a bound on length (default: read from the device)"""
    sfx = _sfx(cache, out)
    assert cache.dim() == 3 and cache.is_contiguous() and cache.shape[2] == 3 * H * D and out.stride(1) == 1
    B = out.shape[0]
    _i32_rows(slot, length, n=B)
    if max_len is None:
        max_len = int(length.max())
    d = H * D
    ld = cache.stride(1)
    base = cache.data_ptr()
    _lib.launches += 1
    call("vsb_attn_decode_slots", base, base + 2 * d, base + 4 * d, out.data_ptr(), cache.stride(0), ld, out.stride(0), B, H, D,
         float(scale), slot.data_ptr(), length.data_ptr(), int(max_len), _DTYPE[sfx], _stream())
    return out


def _gemm_out(a, M, n_out, out, out_dtype, out_rows, residual):
    if out is None:
        out = torch.empty((out_rows if out_rows is not None else M, n_out), dtype=out_dtype or a.dtype, device=a.device)
    _chk(out)
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape[1] >= n_out
    if out.dtype != torch.float32:
        _sfx(a, out)
    if residual is not None:
        _chk(residual, out.dtype)
        assert residual.stride(1) == 1
    return out


def gemm(a, w, out=None, bias=None, residual=None, epilogue=EPI_NONE, out_dtype=None, rows_per_group=0,
         group_stride=0, group_offset=0, out_rows=None, deq_scratch=None):
    """out = epi(a @ w.T + bias) (+ residual).  a [M,K], w [N,K] bf16 or fp16 (row stride arbitrary, inner stride 1); out is
    fp32 or the operands' dtype (default).  w may be an NF4Weight (fp16 a): vsb_gemm_nf4, with deq_scratch (fp16, N*K
    elements) allocated here unless given."""
    nf4 = isinstance(w, NF4Weight)
    if nf4:
        _sfx(a, bias)
        _chk(a, F16)
        N, K2 = w.shape
        fn, w_args = "vsb_gemm_nf4", (w.codes.data_ptr(), w.scales.data_ptr())
    else:
        fn = "vsb_gemm_" + _sfx(a, w, bias)
        pw, N, K2, ldw = _rows2d(w)
        w_args = (pw, ldw)
    pa, M, K, lda = _rows2d(a)
    assert K == K2, (a.shape, w.shape)
    out = _gemm_out(a, M, N // 2 if epilogue == EPI_SWIGLU else N, out, out_dtype, out_rows, residual)
    if bias is not None:
        assert bias.numel() == N and bias.is_contiguous()
    deq = ()
    if nf4:
        if deq_scratch is None:
            deq_scratch = torch.empty((N * K,), dtype=F16, device=a.device)
        _chk(deq_scratch, F16)
        assert deq_scratch.is_contiguous() and deq_scratch.numel() >= N * K
        deq = (deq_scratch.data_ptr(),)
    _lib.launches += 1
    call(fn, pa, lda, *w_args, out.data_ptr(), out.stride(0), M, N, K, _p(bias), _p(residual),
         residual.stride(0) if residual is not None else 0, epilogue, 1 if out.dtype == torch.float32 else 0, rows_per_group, group_stride,
         group_offset, *deq, _stream())
    return out


def gemm_rowscale(a, w, out, rowsq_in=None, rowsq_out=None, eps=1e-6, residual=None, epilogue=EPI_NONE):
    """out = epi(rstd[m] * (a @ w.T)) (+ residual) with the RMSNorm weight already folded into w; rowsq_in fp32 [chunks, M] partial
    sums of squares of a's rows, rowsq_out fp32 [N/32, M] receives those of the stored output (see vsb_gemm_rowscale_bf16)"""
    sfx = _sfx(a, w, out, residual)
    pa, M, K, lda = _rows2d(a)
    pw, N, K2, ldw = _rows2d(w)
    assert K == K2 and out.stride(1) == 1
    for t in (rowsq_in, rowsq_out):
        assert t is None or (t.dtype == torch.float32 and t.is_cuda and t.is_contiguous() and t.shape[1] == M)
    _lib.launches += 1
    call("vsb_gemm_rowscale_" + sfx, pa, lda, pw, ldw, out.data_ptr(), out.stride(0), M, N, K, 0, _p(residual),
         residual.stride(0) if residual is not None else 0, epilogue, 0, 0, 0, _p(rowsq_in), rowsq_in.shape[0] if rowsq_in is not None else 0,
         float(eps), _p(rowsq_out), M, _stream())
    return out


def rowsq(x):
    """fp32 [1, rows] sums of squares of the rows of x (bf16 / fp16)"""
    sfx = _sfx(x)
    px, rows, cols, ldx = _rows2d(x)
    out = torch.empty((1, rows), dtype=torch.float32, device=x.device)
    _lib.launches += 1
    call("vsb_rowsq_" + sfx, px, ldx, out.data_ptr(), rows, cols, _stream())
    return out


def layernorm(x, w, b, eps, out=None, act=EPI_NONE):
    sfx = _sfx(x, w, b, out)
    px, rows, cols, ldx = _rows2d(x)
    if out is None:
        out = torch.empty((rows, cols), dtype=x.dtype, device=x.device)
    _lib.launches += 1
    call("vsb_layernorm_" + sfx, px, ldx, w.data_ptr(), b.data_ptr(), out.data_ptr(), out.stride(0), rows, cols, float(eps), act, _stream())
    return out


def rmsnorm(x, w, eps, out=None):
    sfx = _sfx(x, w, out)
    px, rows, cols, ldx = _rows2d(x)
    if out is None:
        out = torch.empty((rows, cols), dtype=x.dtype, device=x.device)
    _lib.launches += 1
    call("vsb_rmsnorm_" + sfx, px, ldx, w.data_ptr(), out.data_ptr(), out.stride(0), rows, cols, float(eps), _stream())
    return out


def rope_(qkv, T, H, D, cos_t, sin_t, pos0=0, positions=None, rows=None, group_stride=None, group_offset=0):
    """In place on the q|k thirds of qkv [.., 3*H*D].  Default: `rows` = all rows, contiguous groups of T.
    KV-cache layout: logical row r -> physical row (r // T) * group_stride + group_offset + r % T."""
    sfx = _sfx(qkv, cos_t, sin_t)
    p, nrows, cols, ld = _rows2d(qkv)
    assert cols == 3 * H * D
    if rows is None:
        rows = nrows
    if group_stride is None:
        group_stride = T
    _lib.launches += 1
    call("vsb_rope_" + sfx, p, ld, rows, T, H, D, pos0, cos_t.data_ptr(), sin_t.data_ptr(), _p(positions), group_stride, group_offset,
         _stream())
    return qkv


def embed_splice(ids, table, out, img_pos, n_img):
    B, L = ids.shape
    assert ids.dtype == torch.int64 and ids.is_contiguous() and out.is_contiguous()
    _lib.launches += 1
    call("vsb_embed_splice_bf16", ids.data_ptr(), table.data_ptr(), out.data_ptr(), B, L, img_pos, n_img, table.shape[1], table.shape[0], _stream())
    return out


def gather_rows(idx, table, out=None):
    """out[i] = table[idx[i]] (2-byte elements: bf16 or fp16)"""
    assert idx.dtype == torch.int64 and idx.is_contiguous()
    pt, nrows, d, ldt = _rows2d(table)
    n = idx.numel()
    if out is None:
        out = torch.empty((n, d), dtype=table.dtype, device=table.device)
    assert table.element_size() == 2 and out.element_size() == 2
    _lib.launches += 1
    call("vsb_gather_rows_bf16", idx.data_ptr(), pt, ldt, out.data_ptr(), out.stride(0), n, d, nrows, _stream())
    return out


def patchify(pixels, P, Kpad):
    """pixels [B,3,S,S] bf16 / fp16 -> [B*g*g, Kpad] of the same dtype (a 2-byte copy)"""
    _sfx(pixels)
    B, C, S, S2 = pixels.shape
    assert C == 3 and S == S2 and pixels.is_contiguous()
    g = S // P
    out = torch.empty((B * g * g, Kpad), dtype=pixels.dtype, device=pixels.device)
    _lib.launches += 1
    call("vsb_patchify_bf16", pixels.data_ptr(), out.data_ptr(), B, S, P, Kpad, _stream())
    return out


def vit_add_pos_(x, cls, pos, B, S):
    sfx = _sfx(x, cls, pos)
    assert x.is_contiguous()
    _lib.launches += 1
    call("vsb_vit_add_pos_" + sfx, x.data_ptr(), cls.data_ptr(), pos.data_ptr(), B, S, x.shape[-1], _stream())
    return x


def owl_merge(x, w1, b1, w2, b2, B, S, eps):
    C = x.shape[-1]
    assert x.is_contiguous()
    out = torch.empty((B * (S - 1), C), dtype=BF16, device=x.device)
    _lib.launches += 1
    call("vsb_owl_merge_bf16", x.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(), out.data_ptr(), B, S, C, float(eps), _stream())
    return out


def add_rows(a, b, out=None):
    """out[r] = a[r] + b[r % b.rows] (bf16 / fp16)."""
    sfx = _sfx(a, b, out)
    assert a.is_contiguous() and b.is_contiguous() and a.shape[-1] == b.shape[-1]
    a2, b2 = a.view(-1, a.shape[-1]), b.view(-1, b.shape[-1])
    if out is None:
        out = torch.empty_like(a)
    _lib.launches += 1
    call("vsb_add_rows_" + sfx, a2.data_ptr(), b2.data_ptr(), out.data_ptr(), a2.shape[0], a2.shape[1], b2.shape[0], _stream())
    return out


def cast_f32_bf16(x):
    return cast_f32(x, BF16)


def cast_f32(x, dtype, out=None):
    """fp32 -> bf16 / fp16 copy of x (round to nearest even), into `out` (contiguous, same shape) if given"""
    _chk(x, torch.float32)
    assert x.is_contiguous()
    if dtype not in _SUFFIX:
        raise _lib.VsbError(f"unsupported dtype {dtype}: the kernels take bf16 or fp16")
    if out is None:
        out = torch.empty(x.shape, dtype=dtype, device=x.device)
    _chk(out, dtype)
    assert out.is_contiguous() and out.shape == x.shape
    _lib.launches += 1
    call("vsb_cast_f32_" + _SUFFIX[dtype], x.data_ptr(), out.data_ptr(), x.numel(), _stream())
    return out


def argmax_rows(x, out=None):
    """fp32 x [rows, n] (unit inner stride) -> (idx int32 [rows], val fp32 [rows] = x[row, idx]), the index torch.argmax
    returns: the first maximum, where NaN counts as larger than every number (the first NaN wins).  out: idx buffer"""
    _chk(x, torch.float32)
    p, rows, n, ld = _rows2d(x)
    idx = _idx_out(out, rows, x.device)
    val = torch.empty((rows,), dtype=torch.float32, device=x.device)
    _lib.launches += 1
    call("vsb_argmax_rows_f32", p, ld, rows, n, idx.data_ptr(), val.data_ptr(), _stream())
    return idx, val


def _idx_out(out, rows, device):
    if out is None:
        return torch.empty((rows,), dtype=torch.int32, device=device)
    assert out.dtype == torch.int32 and out.shape == (rows,) and out.is_contiguous()
    return out


def sample_rows(x, temperature, top_k, top_p, dtype, seeds, step):
    """one sampled token per row of fp32 logits x [rows, n] (vsb_sample_rows_f32): the logits rounded to `dtype` (bf16 / fp16)
    and divided by `temperature` (> 0), top_k (0 = off, ties at the k-th value kept), top_p (None or 1 = off), then an
    inverse-CDF draw keyed by seeds (int64 [rows] on the device) and `step` -> idx int32 [rows]"""
    _chk(x, torch.float32)
    p, rows, n, ld = _rows2d(x)
    _chk(seeds, torch.int64)
    assert seeds.numel() == rows and seeds.is_contiguous()
    if dtype not in _SUFFIX:
        raise _lib.VsbError(f"unsupported dtype {dtype}: the logits are rounded to bf16 or fp16")
    idx = torch.empty((rows,), dtype=torch.int32, device=x.device)
    _lib.launches += 1
    call("vsb_sample_rows_f32", p, ld, rows, n, float(temperature), int(top_k), 1.0 if top_p is None else float(top_p),
         1 if dtype == F16 else 0, seeds.data_ptr(), int(step), idx.data_ptr(), _stream())
    return idx


def sample_rows_var(x, temperature, top_k, top_p, dtype, seeds, steps, out=None):
    """sample_rows with every row's own settings (vsb_sample_rows_var_f32): temperature fp32, top_k int32 (0 = off), top_p
    fp32 (1 = off), seeds int64 and steps int32, each [rows] on the device -> idx int32 [rows] (or into `out`).  The settings
    are not checked on the device: the caller validates them (vqa.check_sampling, temperature > 0)."""
    _chk(x, torch.float32)
    p, rows, n, ld = _rows2d(x)
    for t, dt in ((temperature, torch.float32), (top_k, torch.int32), (top_p, torch.float32), (seeds, torch.int64), (steps, torch.int32)):
        _chk(t, dt)
        assert t.shape == (rows,) and t.is_contiguous()
    if dtype not in _SUFFIX:
        raise _lib.VsbError(f"unsupported dtype {dtype}: the logits are rounded to bf16 or fp16")
    idx = _idx_out(out, rows, x.device)
    _lib.launches += 1
    call("vsb_sample_rows_var_f32", p, ld, rows, n, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), 1 if dtype == F16 else 0,
         seeds.data_ptr(), steps.data_ptr(), idx.data_ptr(), _stream())
    return idx


BEAM_MAX = 16                                   # VSB_BEAM_MAX
COPY_ROWS_MAX_PAIRS = 256                       # VSB_COPY_ROWS_MAX_PAIRS
SWAP_PAGES_PER_LAUNCH = 384                     # VSB_SWAP_PAGES_PER_LAUNCH


def beam_candidates(x, rows, scores, k, dtype, out=None):
    """one beam-search step (vsb_beam_candidates_f32) for R requests: x fp32 logits [*, V] (unit inner stride), rows int32
    [R, k_in] the rows of x holding each request's beams in beam order, scores fp32 [R, k_in] their running scores (device).
    Log-softmax of the logits rounded to `dtype`, + beam score, the 2k best per request (ties by ascending beam * V + token).
    -> int32 [3, R, 2k]: scores (fp32 bits), tokens, beams - one buffer, so the host reads it with one copy"""
    _chk(x, torch.float32)
    p, _, V, ld = _rows2d(x)
    _chk(rows, torch.int32)
    _chk(scores, torch.float32)
    assert rows.dim() == 2 and rows.is_contiguous() and scores.shape == rows.shape and scores.is_contiguous()
    if dtype not in _SUFFIX:
        raise _lib.VsbError(f"unsupported dtype {dtype}: the logits are rounded to bf16 or fp16")
    R, k_in = rows.shape
    if out is None:
        out = torch.empty((3, R, 2 * k), dtype=torch.int32, device=x.device)
    assert out.shape == (3, R, 2 * k) and out.dtype == torch.int32 and out.is_contiguous()
    _lib.launches += 1
    call("vsb_beam_candidates_f32", p, ld, V, R, k_in, int(k), rows.data_ptr(), scores.data_ptr(), 1 if dtype == F16 else 0,
         out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), _stream())
    return out


def copy_cache_rows(cache, pairs, lo, hi):
    """rows [lo, hi) of every layer of the fused-QKV cache [L, B, Tmax, 3d] from slot s to slot d for every (s, d) in the host
    list `pairs` (vsb_copy_cache_rows_b16, one launch per COPY_ROWS_MAX_PAIRS pairs).  A slot that is both a source and a
    destination raises VsbError."""
    import ctypes
    _chk(cache)
    assert cache.dim() == 4 and cache.element_size() == 2 and cache.stride(3) == 1
    if len(pairs) > COPY_ROWS_MAX_PAIRS:
        srcs = {s for s, _ in pairs}
        if srcs & {d for _, d in pairs}:
            raise _lib.VsbError("vsb_copy_cache_rows_b16: a slot is both a source and a destination")
    L, B, _, W = cache.shape
    for i in range(0, max(1, len(pairs)), COPY_ROWS_MAX_PAIRS):
        chunk = pairs[i:i + COPY_ROWS_MAX_PAIRS]
        arr = (ctypes.c_int * (2 * max(1, len(chunk))))(*[v for pr in chunk for v in pr])
        _lib.launches += 1
        call("vsb_copy_cache_rows_b16", cache.data_ptr(), L, cache.stride(0), B, cache.stride(1), cache.stride(2), W, arr, len(chunk),
             int(lo), int(hi), _stream())
    return cache


def copy_slot_rows(cache, quads):
    """copy_cache_rows with a row range per pair: rows [lo, hi) of every layer from slot s to slot d for every (s, d, lo, hi) in
    the host list `quads`, in one vsb_copy_slot_rows_b16 launch (at most COPY_ROWS_MAX_PAIRS pairs).  A slot that is both a
    source and a destination, a destination named twice, a slot outside the cache or lo > hi raises VsbError."""
    import ctypes
    _chk(cache)
    assert cache.dim() == 4 and cache.element_size() == 2 and cache.stride(3) == 1
    L, B, _, W = cache.shape
    arr = (ctypes.c_int * (4 * max(1, len(quads))))(*[int(v) for q in quads for v in q])
    _lib.launches += 1
    call("vsb_copy_slot_rows_b16", cache.data_ptr(), L, cache.stride(0), B, cache.stride(1), cache.stride(2), W, arr, len(quads), _stream())
    return cache


def nll_rows(logits, labels):
    """logits fp32 [rows, V], labels int64 [rows] -> nll fp32 [rows]"""
    _chk(logits, torch.float32)
    p, rows, n, ld = _rows2d(logits)
    assert labels.dtype == torch.int64 and labels.numel() == rows and labels.is_contiguous()
    out = torch.empty((rows,), dtype=torch.float32, device=logits.device)
    _lib.launches += 1
    call("vsb_nll_rows_f32", p, ld, rows, n, labels.data_ptr(), out.data_ptr(), _stream())
    return out


def copy2d(src, dst):
    """dst[:, :] = src[:, :] for 2-byte element 2-D views with unit inner stride."""
    ps, rows, cols, lds = _rows2d(src)
    pd, rows2, cols2, ldd = _rows2d(dst)
    assert rows == rows2 and cols == cols2 and src.element_size() == 2 and dst.element_size() == 2
    _lib.launches += 1
    call("vsb_copy2d_b16", ps, lds, pd, ldd, rows, cols, _stream())
    return dst


def flash_attn(q, k, v, out, B, H, Sq, Sk, D, causal, scale, q_bs, q_rs, k_bs, k_rs, v_bs, v_rs, o_bs, o_rs):
    """Strided attention: element (b,s,h,d) of q at q.data_ptr() + (b*q_bs + s*q_rs + h*D + d) elements, etc."""
    sfx = _sfx(q, k, v, out)
    _lib.launches += 1
    call("vsb_flash_attn_" + sfx, q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), q_bs, q_rs, k_bs, k_rs, v_bs, v_rs,
         o_bs, o_rs, B, H, Sq, Sk, D, 1 if causal else 0, float(scale), _stream())
    return out


def attn_fused_qkv(qkv, B, S, H, D, causal, scale, out=None):
    """qkv [B*S, 3*H*D] (q|k|v) -> out [B*S, H*D]"""
    ld = qkv.stride(0)
    if out is None:
        out = torch.empty((B * S, H * D), dtype=qkv.dtype, device=qkv.device)
    q = qkv
    k = qkv[:, H * D:]
    v = qkv[:, 2 * H * D:]
    return flash_attn(q, k, v, out, B, H, S, S, D, causal, scale, S * ld, ld, S * ld, ld, S * ld, ld, S * out.stride(0), out.stride(0))


def attn_small(q, k, v, B, H, Nq, Nk, D, scale, out=None):
    sfx = _sfx(q, k, v, out)
    pq, rq, cq, ldq = _rows2d(q)
    pk, rk, ck, ldk = _rows2d(k)
    pv, rv, cv, ldv = _rows2d(v)
    if out is None:
        out = torch.empty((B * Nq, H * D), dtype=q.dtype, device=q.device)
    _lib.launches += 1
    call("vsb_attn_small_" + sfx, pq, ldq, pk, ldk, pv, ldv, out.data_ptr(), out.stride(0), B, H, Nq, Nk, D, float(scale), _stream())
    return out


def owl_class_post(y, query, rows_per_crop, Q, quant_bf16=False):
    """quant_bf16: round logits / scores to bf16 values (what the reference's bf16 model emits), fp32 storage"""
    _chk(y, torch.float32), _chk(query, BF16)
    R = y.shape[0]
    logits = torch.empty((R,), dtype=torch.float32, device=y.device)
    scores = torch.empty((R,), dtype=torch.float32, device=y.device)
    _lib.launches += 1
    call("vsb_owl_class_post", y.data_ptr(), y.stride(0), query.data_ptr(), query.stride(0), rows_per_crop, R, Q, 1 if quant_bf16 else 0,
         logits.data_ptr(), scores.data_ptr(), _stream())
    return logits, scores


def owl_box_post(y, box_bias, rows_per_crop, quant_bf16=False):
    _chk(y, torch.float32), _chk(box_bias, torch.float32)
    R = y.shape[0]
    boxes = torch.empty((R, 4), dtype=torch.float32, device=y.device)
    _lib.launches += 1
    call("vsb_owl_box_post", y.data_ptr(), y.stride(0), box_bias.data_ptr(), rows_per_crop, R, 1 if quant_bf16 else 0, boxes.data_ptr(),
         _stream())
    return boxes


def pack_detections(scores, boxes, rec, row0=0):
    """scores fp32 [n,P], boxes fp32 [n,P,4] -> records rec[row0 : row0+n] (fields 0..7 and 12..75, see records.py)"""
    _chk(scores, torch.float32), _chk(boxes, torch.float32), _chk(rec, torch.float32)
    n, P = scores.shape
    assert scores.is_contiguous() and boxes.is_contiguous() and boxes.shape == (n, P, 4)
    assert rec.dim() == 2 and rec.is_contiguous() and row0 + n <= rec.shape[0]
    _lib.launches += 1
    call("vsb_pack_detections_f32", scores.data_ptr(), boxes.data_ptr(), n, P, rec.data_ptr() + row0 * rec.shape[1] * 4, rec.shape[1],
         _stream())
    return rec


def heat_pyramids(jobs, rec, LH, LW):
    """jobs: list of (low_res fp32 [LH,LW] device view, h, w, rects [(x,y,w,h) relative to the crop], record row).
    Fills the heat-map statistics and rectangle sums of those records straight from the low-res masks (no H x W map)."""
    import numpy as np
    if not jobs:
        return rec
    _chk(rec, torch.float32)
    R = rec.shape[1]
    nj = len(jobs)
    total = sum(len(j[3]) for j in jobs)
    table = np.zeros(nj * 8 + total * 5, dtype=np.int32)
    jt = table[:nj * 8].reshape(nj, 8)
    rt = table[nj * 8:nj * 8 + total * 4].reshape(total, 4)
    rj = table[nj * 8 + total * 4:]
    off = 0
    for k, (low, h, w, rects, row) in enumerate(jobs):
        assert low.dtype == torch.float32 and low.is_cuda and low.is_contiguous() and low.shape[-2:] == (LH, LW)
        assert len(rects) <= R - 76, (len(rects), R)
        p = low.data_ptr()
        jt[k] = (0, 0, h, w, off, len(rects), row, 0)
        jt[k, 0:2] = np.array([p], dtype=np.uint64).view(np.int32)
        if rects:
            rt[off:off + len(rects)] = np.asarray(rects, dtype=np.int32)
            rj[off:off + len(rects)] = k
        off += len(rects)
    dev = rec.device
    tab = torch.from_numpy(table).to(dev, non_blocking=True)
    stats_scratch = torch.empty((nj * 64 * 3,), dtype=torch.float32, device=dev)
    rect_scratch = torch.empty((max(1, total) * 64,), dtype=torch.float64, device=dev)
    base = tab.data_ptr()
    _lib.launches += 2 + (2 if total else 0)
    call("vsb_heat_pyramids_f32", base, nj, base + nj * 32, base + nj * 32 + total * 16, total, LH, LW, rec.data_ptr(), R,
         stats_scratch.data_ptr(), rect_scratch.data_ptr(), _stream())
    return rec


def upsample2x_nhwc(x, B, H, W, C):
    assert x.is_contiguous()
    out = torch.empty((B * 4 * H * W, C), dtype=BF16, device=x.device)
    _lib.launches += 1
    call("vsb_upsample2x_nhwc_bf16", x.data_ptr(), out.data_ptr(), B, H, W, C, _stream())
    return out


def im2col3x3_nhwc(x, B, H, W, C):
    assert x.is_contiguous()
    out = torch.empty((B * H * W, 9 * C), dtype=BF16, device=x.device)
    _lib.launches += 1
    call("vsb_im2col3x3_nhwc_bf16", x.data_ptr(), out.data_ptr(), B, H, W, C, _stream())
    return out


def mask_dot(up, hyper, B, P, C):
    assert up.is_contiguous() and hyper.is_contiguous()
    out = torch.empty((B, P), dtype=torch.float32, device=up.device)
    _lib.launches += 1
    call("vsb_mask_dot_bf16", up.data_ptr(), hyper.data_ptr(), out.data_ptr(), B, P, C, _stream())
    return out


HEATMAP_MAX_BLOCKS = 1184


def heatmap(low, h, w, clamp=True, with_stats=True, out=None):
    """low [LH,LW] fp32 -> (map [h,w] fp32, stats [3] = max,min,sum)"""
    _chk(low, torch.float32)
    assert low.is_contiguous() and low.dim() == 2
    if out is None:
        out = torch.empty((h, w), dtype=torch.float32, device=low.device)
    stats = scratch = None
    if with_stats:
        stats = torch.empty((3,), dtype=torch.float32, device=low.device)
        scratch = torch.empty((3 * HEATMAP_MAX_BLOCKS,), dtype=torch.float32, device=low.device)
    _lib.launches += 2 if with_stats else 1
    call("vsb_heatmap_bilinear_f32", low.data_ptr(), low.shape[0], low.shape[1], out.data_ptr(), h, w, 1 if clamp else 0,
         _p(scratch), _p(stats), _stream())
    return out, stats


def rect_sums(hm, rects, stats):
    """hm [h,w] fp32, rects int32 [n,4] (x,y,w,h), stats [3] -> float64 [n] sums of the normalised map"""
    assert rects.dtype == torch.int32 and rects.is_contiguous()
    n = rects.shape[0]
    out = torch.empty((n,), dtype=torch.float64, device=hm.device)
    scratch = torch.empty((64 * n,), dtype=torch.float64, device=hm.device)
    _lib.launches += 2
    call("vsb_rect_sums_f32", hm.data_ptr(), hm.shape[0], hm.shape[1], rects.data_ptr(), n, stats.data_ptr(), out.data_ptr(),
         scratch.data_ptr(), _stream())
    return out
