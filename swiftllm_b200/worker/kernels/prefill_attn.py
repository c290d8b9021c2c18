"""Reference: swiftllm/worker/kernels/prefill_attn.py (prefill_attention :102-139); also replaces the
vllm_flash_attn.flash_attn_varlen_func call at swiftllm/worker/layers/transformer_layer.py:86-96."""
import torch

from swiftllm_b200 import _lib
from swiftllm_b200.worker.infer_state import LlamaInferState


def prefill_attention(
    q: torch.Tensor,    # [num_prefill_tokens, num_q_heads, head_dim]
    k: torch.Tensor,    # [num_prefill_tokens, num_kv_heads, head_dim]
    v: torch.Tensor,    # [num_prefill_tokens, num_kv_heads, head_dim]
    o: torch.Tensor,    # [num_prefill_tokens, num_q_heads, head_dim]
    model_config,
    engine_config,
    infer_state: LlamaInferState,
):
    assert o.is_contiguous()
    qs, ks, vs = _lib.row_stride(q), _lib.row_stride(k), _lib.row_stride(v)
    _lib.require_device(q)
    Tp, nq, D = q.shape
    nkv = k.shape[1]
    if infer_state.num_prefill_seqs == 0:
        return
    _lib.check(_lib.lib().sllm_prefill_attention(
        q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
        infer_state.prefill_seq_start_locs.data_ptr(), infer_state.prefill_seq_lens.data_ptr(),
        infer_state.softmax_scale, infer_state.num_prefill_seqs, infer_state.max_prefill_len, Tp, nq, nkv, D, qs, ks, vs,
        _lib.dtype_tag(q.dtype), _lib.stream()), "prefill_attention")


def prefill_attention_paged(
    q: torch.Tensor,            # [num_prefill_tokens, num_q_heads, head_dim]  (the chunks' queries, packed)
    k_cache: torch.Tensor,      # [num_blocks, num_layers, num_kv_heads, block_size, head_dim]
    v_cache: torch.Tensor,
    block_table: torch.Tensor,  # [max_seqs, max_blocks_per_seq] int32
    o: torch.Tensor,            # [num_prefill_tokens, num_q_heads, head_dim]
    model_config,
    engine_config,
    infer_state: LlamaInferState,
    cur_layer: int,
):
    """Chunked ("prefix-aware") prefill attention (SURVEY.md §8 f-1; no counterpart in the reference, whose prefill attention
    never reads the KV cache): the chunk's queries sit at positions prefill_prefix_lens[i] + t of their sequence and attend
    to positions <= their own, keys / values read from the paged cache (the chunk's own K/V are stored first)."""
    assert o.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous() and block_table.is_contiguous()
    assert block_table.dtype == torch.int32 and infer_state.seq_ids.dtype == torch.int32
    prefix = infer_state.prefill_prefix_lens
    assert prefix is not None and prefix.dtype == torch.int32 and prefix.is_contiguous()
    qs = _lib.row_stride(q)
    _lib.require_device(q)
    Tp, nq, D = q.shape
    if infer_state.num_prefill_seqs == 0:
        return
    num_blocks, num_layers, nkv, bs, _ = k_cache.shape
    _lib.check(_lib.lib().sllm_prefill_attention_paged(
        q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(), block_table.data_ptr(),
        infer_state.seq_ids.data_ptr(), infer_state.prefill_seq_start_locs.data_ptr(), infer_state.prefill_seq_lens.data_ptr(),
        prefix.data_ptr(), infer_state.softmax_scale, infer_state.num_prefill_seqs, infer_state.max_prefill_len, Tp,
        cur_layer, num_layers, nq, nkv, bs, D, block_table.shape[1], num_blocks, qs,
        _lib.dtype_tag(q.dtype), _lib.stream()), "prefill_attention_paged")


def paged_attention_verify(
    q: torch.Tensor,            # [num_tokens, num_q_heads, head_dim]  (every row of every speculative entry, packed)
    k_cache: torch.Tensor,
    v_cache: torch.Tensor,
    block_table: torch.Tensor,
    o: torch.Tensor,            # [num_tokens, num_q_heads, head_dim]
    model_config,
    engine_config,
    infer_state: LlamaInferState,
    cur_layer: int,
):
    """Speculative verification: prefill_attention_paged's function for entries of 1..8 rows (prefill_seq_lens), computed by
    the multi-query paged kernel that reads each (entry, kv head) page once for all of the entry's rows."""
    assert o.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous() and block_table.is_contiguous()
    assert block_table.dtype == torch.int32 and infer_state.seq_ids.dtype == torch.int32
    prefix = infer_state.prefill_prefix_lens
    assert prefix is not None and prefix.dtype == torch.int32 and prefix.is_contiguous()
    qs = _lib.row_stride(q)
    _lib.require_device(q)
    T, nq, D = q.shape
    if infer_state.num_prefill_seqs == 0:
        return
    num_blocks, num_layers, nkv, bs, _ = k_cache.shape
    l = _lib.lib()
    B, max_len = infer_state.num_prefill_seqs, infer_state.max_prefill_kv_len
    ws_bytes = l.sllm_paged_attention_verify_workspace_bytes(B, T, nq, nkv, D, max_len)
    ws = torch.empty((ws_bytes // 4,), dtype=torch.float32, device=q.device) if ws_bytes > 0 else None
    _lib.check(l.sllm_paged_attention_verify(
        q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(), block_table.data_ptr(),
        infer_state.seq_ids.data_ptr(), infer_state.prefill_seq_start_locs.data_ptr(), infer_state.prefill_seq_lens.data_ptr(),
        prefix.data_ptr(), _lib.ptr(ws), ws_bytes, infer_state.softmax_scale, B, infer_state.max_prefill_len, max_len, T,
        cur_layer, num_layers, nq, nkv, bs, D, block_table.shape[1], num_blocks, qs,
        _lib.dtype_tag(q.dtype), _lib.stream()), "paged_attention_verify")
