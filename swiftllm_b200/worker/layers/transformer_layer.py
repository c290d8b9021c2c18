"""One Llama decoder layer.  Op sequence of the reference (swiftllm/worker/layers/transformer_layer.py:31-130):
fused add+RMSNorm -> q/k/v GEMMs -> rotary -> KV store -> attention (prefill: causal varlen flash attention on the
packed prompt tokens; decode: paged attention through the block table) -> o_proj -> fused add+RMSNorm ->
up_gate GEMM -> SiLU*mul -> down GEMM.  q/k/v come from ONE fused GEMM.

Differences by design: the prefill attention is this library's own kernel (the reference calls third-party
vllm_flash_attn, :86-96); with tensor parallelism each rank runs its head / FFN-column shard and the partial
o_proj / down_proj outputs are summed with ONE NCCL all-reduce each (the only collectives of the model); the
side stream for decode attention (:103-114) is only used when the batch really mixes prefill and decode work.

Per-request LoRA adapters (infer_state.lora, worker/lora.py): right after each of the four GEMMs (qkv, o, up_gate, down) a
shrink and an expand launch add the adapters' deltas into the GEMM output in place - under TP into the rank's partial output
(the NCCL buffer or comm.partial_out) before the exchange sums the ranks.

FP8 weights (weight.fp8, worker/fp8.py): the same sequence with e4m3 GEMM inputs.  The kernels that produce each input quantize it
per token (csrc/fp8.cu) and the GEMMs are the library's row-wise scaled FP8 GEMM (linear_fp8): add+RMSNorm+quantize -> qkv ->
rotary / KV store / attention as above -> quantize -> o_proj -> add+RMSNorm+quantize (or the exchange, then quantize) -> up_gate
-> SiLU*mul+quantize -> down_proj.  Under TP the row-parallel inputs are quantized per rank on the rank's K slice.
"""
import torch
import torch.distributed as dist

from swiftllm_b200.worker.infer_state import LlamaInferState
from swiftllm_b200.worker.kernels.kvcache_mgmt import rotary_store_kvcache_decode, store_kvcache
from swiftllm_b200.worker.kernels.fp8 import fused_add_rmsnorm_quant_fp8, quant_fp8_rows, silu_and_mul_quant_fp8
from swiftllm_b200.worker.kernels.linear import linear, linear_fp8
from swiftllm_b200.worker.kernels.lora import lora_expand, lora_shrink
from swiftllm_b200.worker.kernels.paged_attn import paged_attention
from swiftllm_b200.worker.kernels.prefill_attn import paged_attention_verify, prefill_attention, prefill_attention_paged
from swiftllm_b200.worker.kernels.rmsnorm import fused_add_rmsnorm_inplace
from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
from swiftllm_b200.worker.kernels.silu_and_mul import silu_and_mul_inplace


class LlamaTransformerLayer:
    def __init__(self, model_config, engine_config, weight, decoding_piggyback_stream, layer_id: int,
                 tp_group=None, comm=None):
        self.model_config = model_config
        self.engine_config = engine_config
        self.weight = weight
        self.decoding_piggyback_stream = decoding_piggyback_stream
        self.layer_id = layer_id
        self.tp_size = getattr(engine_config, "tp_size", 1)
        self.tp_group = tp_group
        self.fuse_rotary_store = bool(getattr(engine_config, "fuse_rotary_store", True))
        self.comm = comm            # FusedAllReduce (tp_comm.py) or None -> NCCL all-reduce + separate add/norm kernels
        self.num_q_heads = model_config.num_q_heads // self.tp_size      # per-rank shard
        self.num_kv_heads = model_config.num_kv_heads // self.tp_size
        self.ffn_inter_dim = model_config.ffn_inter_dim // self.tp_size

    def _all_reduce(self, x: torch.Tensor):
        if self.tp_size > 1:
            dist.all_reduce(x, group=self.tp_group)

    def _lora(self, lora, site: int, x: torch.Tensor, y: torch.Tensor):
        """y += the step's adapter deltas at `site` (worker.lora.SITES index); nothing when the step has no adapter."""
        if lora is None:
            return
        p = lora.pool
        mask = p.slice_mask[self.layer_id, site]
        lora_shrink(x, p.u, p.a[self.layer_id][site], lora.tiles, mask)
        lora_expand(y, p.u, p.b[self.layer_id][site], p.dims_ends[site], lora.tiles, mask, p.scales)

    def _attention(self, qkv: torch.Tensor, input_embds: torch.Tensor, k_cache, v_cache, block_table,
                   infer_state: LlamaInferState) -> torch.Tensor:
        """Rotary, KV store and attention of the qkv GEMM output; the attention output [T, nq * D] (at TP 1 written over
        input_embds, which the GEMM has consumed)."""
        mc = self.model_config
        T, nqd, nkvd = qkv.shape[0], self.num_q_heads * mc.head_dim, self.num_kv_heads * mc.head_dim
        q = qkv[:, :nqd].unflatten(1, (self.num_q_heads, mc.head_dim))
        k = qkv[:, nqd:nqd + nkvd].unflatten(1, (self.num_kv_heads, mc.head_dim))
        v = qkv[:, nqd + nkvd:].unflatten(1, (self.num_kv_heads, mc.head_dim))

        if self.fuse_rotary_store and infer_state.num_prefill_seqs == 0 and not infer_state.ignore_kvcache:
            # pure decode: rotary + KV store of the new rows in one launch
            rotary_store_kvcache_decode(q, k, v, k_cache, v_cache, block_table, infer_state, self.layer_id)
        else:
            rotary_embedding_inplace(q, k, infer_state)
            if not infer_state.ignore_kvcache:
                store_kvcache(k, v, k_cache, v_cache, block_table, mc, self.engine_config, infer_state, self.layer_id)

        npt = infer_state.num_prefill_tokens
        o = input_embds if self.tp_size == 1 else torch.empty((q.shape[0], self.num_q_heads * mc.head_dim),
                                                               dtype=q.dtype, device=q.device)
        mixed = infer_state.num_prefill_seqs > 0 and infer_state.num_decoding_seqs > 0
        if mixed:
            store_kvcache_event = torch.cuda.Event()
            store_kvcache_event.record()
        if infer_state.num_prefill_seqs > 0:
            if infer_state.prefill_prefix_lens is not None:
                # chunked prefill: attend to prefix + chunk through the block table (the chunk's K/V were stored above)
                attend = paged_attention_verify if infer_state.speculative else prefill_attention_paged
                attend(q[:npt], k_cache, v_cache, block_table, o[:npt].view(npt, self.num_q_heads, mc.head_dim), mc,
                       self.engine_config, infer_state, self.layer_id)
            else:
                prefill_attention(q[:npt], k[:npt], v[:npt], o[:npt].view(npt, self.num_q_heads, mc.head_dim),
                                  mc, self.engine_config, infer_state)
        if infer_state.num_decoding_seqs > 0:
            assert not infer_state.ignore_kvcache
            if mixed:
                with torch.cuda.stream(self.decoding_piggyback_stream):
                    torch.cuda.current_stream().wait_event(store_kvcache_event)
                    paged_attention(q[npt:], k_cache, v_cache, block_table, mc, self.engine_config, infer_state,
                                    self.layer_id, o[npt:])
                    event = torch.cuda.Event()
                    event.record()
                torch.cuda.current_stream().wait_event(event)
            else:
                paged_attention(q[npt:], k_cache, v_cache, block_table, mc, self.engine_config, infer_state,
                                self.layer_id, o[npt:])
        return o

    def forward(
        self,
        input_embds: torch.Tensor,  # [num_tokens, hidden_size]
        residual_buf: torch.Tensor,  # [num_tokens, hidden_size]
        k_cache: torch.Tensor,
        v_cache: torch.Tensor,
        block_table: torch.Tensor,
        infer_state: LlamaInferState,
    ) -> torch.Tensor:
        mc, w = self.model_config, self.weight
        # fused exchange (tp_comm.py) for steps it covers; the same choice in every layer of a step (the row count is fixed)
        comm = self.comm if (self.comm is not None and residual_buf.shape[0] <= self.comm.max_fused_tokens) else None
        if w.fp8:
            return self._forward_fp8(input_embds, residual_buf, k_cache, v_cache, block_table, infer_state, comm)
        if comm is not None and self.layer_id > 0:
            # the previous layer left its down_proj PARTIAL in symmetric buffer 1: exchange + add + norm in one kernel
            input_embds = comm.reduce_add_norm(1, residual_buf.shape[0], residual_buf, w.attn_norm, mc.rms_norm_eps)
        else:
            fused_add_rmsnorm_inplace(input_embds, residual_buf, w.attn_norm, mc.rms_norm_eps)

        # one GEMM for q, k and v (three latency-bound GEMMs in the reference, transformer_layer.py:54-56); the
        # kernels below take the row-strided column slices directly
        qkv = linear(input_embds, w.qkv_proj)
        lora = infer_state.lora
        self._lora(lora, 0, input_embds, qkv)
        o = self._attention(qkv, input_embds, k_cache, v_cache, block_table, infer_state)

        if comm is not None:
            T = o.shape[0]
            torch.mm(o, w.o_proj.t(), out=comm.partial_out(0, T))              # partial sums -> symmetric buffer 0
            self._lora(lora, 1, o, comm.partial_out(0, T))
            o = comm.reduce_add_norm(0, T, residual_buf, w.ffn_norm, mc.rms_norm_eps)
            up_gate_proj = linear(o, w.up_gate_proj)
            self._lora(lora, 2, o, up_gate_proj)
            silu_and_mul_inplace(up_gate_proj)
            ffn_out = comm.partial_out(1, T)                                   # consumed by the next layer / the model tail
            torch.mm(up_gate_proj[:, :self.ffn_inter_dim], w.down_proj.t(), out=ffn_out)
            self._lora(lora, 3, up_gate_proj[:, :self.ffn_inter_dim], ffn_out)
            return ffn_out

        attn = o
        o = linear(o, w.o_proj)                # row-parallel under TP: partial sums
        self._lora(lora, 1, attn, o)
        self._all_reduce(o)
        fused_add_rmsnorm_inplace(o, residual_buf, w.ffn_norm, mc.rms_norm_eps)

        up_gate_proj = linear(o, w.up_gate_proj)
        self._lora(lora, 2, o, up_gate_proj)
        silu_and_mul_inplace(up_gate_proj)
        ffn_out = linear(up_gate_proj[:, :self.ffn_inter_dim], w.down_proj)
        self._lora(lora, 3, up_gate_proj[:, :self.ffn_inter_dim], ffn_out)
        self._all_reduce(ffn_out)
        return ffn_out

    def _forward_fp8(self, input_embds, residual_buf, k_cache, v_cache, block_table, infer_state, comm):
        mc, w, dt = self.model_config, self.weight, residual_buf.dtype
        if comm is not None and self.layer_id > 0:
            xq, xs = quant_fp8_rows(comm.reduce_add_norm(1, residual_buf.shape[0], residual_buf, w.attn_norm, mc.rms_norm_eps))
        else:
            xq, xs = fused_add_rmsnorm_quant_fp8(input_embds, residual_buf, w.attn_norm, mc.rms_norm_eps)
        qkv = linear_fp8(xq, xs, w.qkv_proj, w.qkv_proj_scale, dt)
        o = self._attention(qkv, input_embds, k_cache, v_cache, block_table, infer_state)
        oq, os_ = quant_fp8_rows(o)
        T = o.shape[0]
        if comm is not None:
            linear_fp8(oq, os_, w.o_proj, w.o_proj_scale, dt, out=comm.partial_out(0, T))   # partial sums -> symmetric buffer 0
            xq, xs = quant_fp8_rows(comm.reduce_add_norm(0, T, residual_buf, w.ffn_norm, mc.rms_norm_eps))
        else:
            o = linear_fp8(oq, os_, w.o_proj, w.o_proj_scale, dt)                          # row-parallel under TP: partial sums
            self._all_reduce(o)
            xq, xs = fused_add_rmsnorm_quant_fp8(o, residual_buf, w.ffn_norm, mc.rms_norm_eps)
        up_gate_proj = linear_fp8(xq, xs, w.up_gate_proj, w.up_gate_proj_scale, dt)
        hq, hs = silu_and_mul_quant_fp8(up_gate_proj)
        ffn_out = linear_fp8(hq, hs, w.down_proj, w.down_proj_scale, dt, out=None if comm is None else comm.partial_out(1, T))
        if comm is None:
            self._all_reduce(ffn_out)
        return ffn_out
