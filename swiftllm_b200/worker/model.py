"""LlamaModel - the data-plane worker.  Same public API as the reference's
`swiftllm.worker.model.LlamaModel` (swiftllm/worker/model.py:18-408):

    LlamaModel(engine_config) -> load_weights() -> profile_num_blocks() -> init_kvcache_and_swap(num_blocks)
    forward(input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache=False) -> list[int]
                                                           (addition: sampling parameters, allowed-token masks)
    forward_with_logprobs(...) -> list[TokenLogprobs]      (addition: forward's arguments, tokens with log-probabilities,
                                                            and of prompt tokens with SamplingParams.prompt_logprobs)
    forward_speculative(input_ids_list, seq_ids_list, prefix_lens_list, sampling_params_list=None) -> list[list[int]]
                                                            (addition: verify up to 7 drafts per sequence in one step)
    fork_seqs(src_seq_ids_list, dst_seq_ids_list, lens_list)  (addition: share a cached prefix with another sequence)
    load_lora(slot, adapter) / unload_lora(slot)               (addition: per-request LoRA adapters, lora_ids_list)
    swap_in_seqs / swap_out_seqs / free_seqs_resources

and the same observable state (k_cache, v_cache, k_swap, v_swap, gpu_block_manager, cpu_block_manager).  Addition: the token
pages token_cache / token_swap (int32 [blocks, block_size], id | is_output << 31), the history the penalty kernel reads.

Host path (SURVEY.md §8 f-2): all per-step metadata travels in ONE pinned staging buffer and one
H2D copy (the reference issues ~6 small copies, model.py:272-297); block allocation is one sync-free kernel
(three syncs + torch.nonzero in the reference, block_manager.py:50,70,75); pure-decode steps can be replayed
from a CUDA graph; the only sync of a step is the final `.tolist()` of the sampled tokens.
"""
from __future__ import annotations

import dataclasses
import itertools
import math
from typing import Callable, Optional

import numpy as np
import torch
import torch.distributed as dist

from swiftllm_b200 import swiftllm_c
from swiftllm_b200.engine_config import EngineConfig
from swiftllm_b200.model_config import LlamaModelConfig
from swiftllm_b200.sampling_params import (ConstraintWords, PromptLogprobs, SamplingParams, TokenLogprobs, constraint_words,
                                           check_breaker_ids, has_ngram_controls, has_penalties, has_truncation, logprobs_top_n,
                                           prompt_logprobs_top_n, sampling_words)
from swiftllm_b200.utils import GB
from swiftllm_b200.worker import fp8 as fp8_weights
from swiftllm_b200.worker.block_manager import BlockManager
from swiftllm_b200.worker.kernels.block_mgmt import copy_block_tails
from swiftllm_b200.worker.lora import LoraPool, lora_tiles
from swiftllm_b200.worker.weight import load_weights

from .infer_state import ConstraintState, LlamaInferState, LoraState, PromptLogprobsState, SamplingState
from .layers.post_layer import LlamaPostLayer
from .layers.pre_layer import LlamaPreLayer
from .layers.transformer_layer import LlamaTransformerLayer

_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def select_seq_block_size(num_kv_heads: int, decoding_seq_lens_list: list, max_decoding_len: int) -> int:
    """The reference's flash-decoding split heuristic, verbatim in behaviour (model.py:305-324)."""
    seq_block_size = 2048
    decoding_seq_lens_sum = sum(decoding_seq_lens_list)
    while num_kv_heads * (decoding_seq_lens_sum / seq_block_size) < 1024 and seq_block_size // 2 >= 64 and \
            max_decoding_len / (seq_block_size // 2) <= 128:
        seq_block_size //= 2
    return seq_block_size


def build_rope_tables(model_config: LlamaModelConfig, dtype: torch.dtype):
    """cos/sin tables [max_seq_len + 128, head_dim/2] (model.py:177-225), computed in fp32 on the HOST so the
    tables are bit-identical on every device and to the CPU oracle, then rounded to the model dtype."""
    rope_scaling = model_config.rope_scaling
    base = model_config.rope_theta
    max_pos = model_config.max_position_embeddings
    dim = model_config.head_dim
    if isinstance(rope_scaling, dict):      # Llama 3.2 style dictionary (model.py:183-211)
        factor = rope_scaling.get("factor", 4.0)
        low = rope_scaling.get("low_freq_factor", 1.0)
        high = rope_scaling.get("high_freq_factor", 1.0)
        orig = rope_scaling.get("original_max_position_embeddings", max_pos)
        max_seq_len = int(orig * factor)
        t = torch.arange(max_seq_len + 128, dtype=torch.float32)
        split = int((dim // 2) * low / (low + high))
        inv_low = 1.0 / (base ** (torch.arange(0, split * 2, 2, dtype=torch.float32) / dim))
        inv_high = 1.0 / (base ** (torch.arange(split * 2, dim, 2, dtype=torch.float32) / dim))
        freqs = torch.cat([torch.outer(t / low, inv_low), torch.outer(t / high, inv_high)], dim=-1)
    else:
        max_seq_len = max_pos * rope_scaling
        inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))
        t = torch.arange(int(max_seq_len + 128), dtype=torch.float32) / rope_scaling
        freqs = torch.outer(t, inv_freq)
    return torch.cos(freqs).to(dtype), torch.sin(freqs).to(dtype)


class LlamaModel:
    @torch.inference_mode()
    def __init__(self, engine_config: EngineConfig, model_config: Optional[LlamaModelConfig] = None):
        """`model_config` may be given directly (synthetic-weight runs); otherwise it is read from
        engine_config.model_path/config.json like the reference (model.py:42)."""
        self.engine_config = engine_config
        self.model_config = model_config if model_config is not None else \
            LlamaModelConfig.load_from_model_path(engine_config.model_path)
        self.dtype = _DTYPES[getattr(engine_config, "dtype", "float16")]
        self.tp_size = getattr(engine_config, "tp_size", 1)
        self.tp_rank = getattr(engine_config, "tp_rank", 0)
        mc = self.model_config
        assert mc.num_q_heads % self.tp_size == 0 and mc.num_kv_heads % self.tp_size == 0 and \
            mc.ffn_inter_dim % self.tp_size == 0, "tp_size must divide q heads, kv heads and ffn_inter_dim"
        # FP8 projections (worker/fp8.py): unsupported formats and combinations raise ValueError before anything is allocated
        self.fp8 = fp8_weights.resolve(getattr(engine_config, "quantization", None), mc, self.tp_size,
                                       getattr(engine_config, "max_loras", 0), self.dtype)
        self.device = torch.device("cuda", torch.cuda.current_device())

        self.weight = None
        self._cos_cached = self._sin_cached = None
        self.pre_layer = None
        self.transformer_layers = None
        self.post_layer = None
        self.num_blocks = None
        self.k_cache = self.v_cache = None
        self.k_swap = self.v_swap = None
        # token pages (SamplingParams penalties and n-gram controls): written in steps with such a row, carried in swaps once
        # one has run
        self.token_cache = self.token_swap = None
        self._penalties_used = False
        self.cpu_block_manager = self.gpu_block_manager = None
        self.tp_group = None
        self.lora = None                # LoraPool (EngineConfig.max_loras > 0)
        self._graphs = {}
        # pinned staging ring for per-step metadata (every step path): a slot is rewritten only after the H2D copy that last read it
        # has completed (event per slot), so back-to-back forward_async calls never race the copy engine
        self._stage_ring = []
        self._stage_next = 0
        self._swap_stream = None        # EngineConfig.swap_on_copy_stream: dedicated copy stream + "copies done" event
        self._swap_done = None
        # seeds of SamplingParams(seed=None) rows: every rank of a tensor-parallel group draws the same sequence
        self._sampling_rng = np.random.default_rng(getattr(engine_config, "sampling_seed", 0))

    # ------------------------------------------------------------------ init
    @torch.inference_mode()
    def load_weights(self, weight_getter: Optional[Callable] = None):
        """Load weights (checkpoint, dummy, or a custom getter(key, shape, dtype) -> full tensor) and build layers."""
        if self.tp_size > 1:
            assert dist.is_initialized(), "tensor parallelism needs torch.distributed (NCCL) to be initialised"
            self.tp_group = dist.group.WORLD
        self.weight = load_weights(self.model_config, self.dtype, self.engine_config.model_path,
                                   self.engine_config.use_dummy, getter=weight_getter,
                                   tp_rank=self.tp_rank, tp_size=self.tp_size, device=self.device,
                                   shard_lm_head=self._shard_lm_head(), fp8=self.fp8)
        cos, sin = build_rope_tables(self.model_config, self.dtype)
        self._cos_cached, self._sin_cached = cos.to(self.device), sin.to(self.device)

        self.comm = None
        want_fused = getattr(self.engine_config, "fused_allreduce", None)
        explicit = want_fused is not None
        if want_fused is None:
            #   tp 2, 4: one-shot peer-memory kernel
            #   tp 8:    row-owner kernel with in-switch reduction and broadcast (falls back to peer memory, then NCCL)
            candidates = [True] if 2 <= self.tp_size <= 4 else (["two_shot_nvls", "two_shot"] if self.tp_size == 8 else [])
        else:
            candidates = [want_fused] if want_fused else []
        for cand in candidates if self.tp_size > 1 else []:
            two_shot = cand in ("two_shot", "two_shot_nvls", "ll", "ll_nvls")      # row-owner exchanges
            nvls = cand in ("two_shot_nvls", "ll_nvls")                            # in-switch reduction / broadcast (multimem)
            ll = cand in ("ll", "ll_nvls")                                         # barrier-free push kernel
            from swiftllm_b200.worker.tp_comm import FusedAllReduce
            comm = None
            try:
                comm = FusedAllReduce(self.engine_config.max_tokens_in_batch, self.model_config.hidden_size,
                                      self.dtype, self.device, self.tp_group, two_shot=two_shot, nvls=nvls, ll=ll)
            except Exception as e:      # noqa: BLE001  (no peer access / symmetric memory / multicast unavailable)
                if explicit:
                    raise
                import warnings
                warnings.warn(f"fused exchange `{cand}` unavailable ({e}); trying the next option")
            # every rank must take the same path
            ok = torch.tensor([1 if comm is not None else 0], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.tp_group)
            if int(ok.item()) == 1:
                self.comm = comm
                break
            del comm
        decoding_piggyback_stream = torch.cuda.Stream()
        self.pre_layer = LlamaPreLayer(self.model_config, self.weight)
        self.transformer_layers = [
            LlamaTransformerLayer(self.model_config, self.engine_config, self.weight.layers[i],
                                  decoding_piggyback_stream, i, tp_group=self.tp_group, comm=self.comm)
            for i in range(self.model_config.num_layers)
        ]
        self.post_layer = LlamaPostLayer(self.model_config, self.weight, tp_group=self.tp_group, tp_rank=self.tp_rank,
                                         tp_size=self.tp_size)
        ec = self.engine_config
        if getattr(ec, "max_loras", 0):
            # allocated before profile_num_blocks, so the KV-cache sizing leaves room for it
            self.lora = LoraPool(self.model_config, ec.max_loras, getattr(ec, "max_lora_rank", 0), self.dtype, self.device,
                                 ec.max_tokens_in_batch, tp_rank=self.tp_rank, tp_size=self.tp_size)
            print(f"[Model.lora] {ec.max_loras} adapter slots of rank {self.lora.rank}: {self.lora.nbytes() / GB:.3f} GB "
                  f"({self.lora.nbytes() / ec.max_loras / 2 ** 20:.1f} MiB per slot)")

    # ------------------------------------------------------------------ LoRA adapters
    @torch.inference_mode()
    def load_lora(self, slot: int, adapter):
        """Copy a PEFT LoRA adapter into slot `slot` (replacing what it held); requests choose it with lora_ids_list.  `adapter`
        is a PEFT adapter directory (adapter_config.json + adapter_model.safetensors or adapter_model.bin) or a (config dict,
        {PEFT key: tensor}) pair.  Read keys: base_model.model.model.layers.{i}.{self_attn,mlp}.{q,k,v,o,gate,up,down}_proj
        .lora_{A,B}.weight, A [r, in], B [out, r]; scale lora_alpha / r (lora_alpha / sqrt(r) with use_rslora); tensors are
        rounded once to the model dtype.  Modules the adapter leaves out keep the base model's outputs bit for bit.  Raises
        ValueError before anything is copied for: max_loras 0, a slot outside [0, max_loras), r > max_lora_rank, a shape that
        does not match the model, fan_in_fan_out, bias other than "none", DoRA, a non-empty rank_pattern / alpha_pattern /
        modules_to_save / layers_to_transform, adapters on embed_tokens or lm_head, and tensors under any other key.  Each
        tensor-parallel rank loads the same adapter and keeps its slices."""
        if self.lora is None:
            raise ValueError("load_lora: the engine has no adapter slots (EngineConfig.max_loras is 0)")
        self.lora.load(slot, adapter)

    @torch.inference_mode()
    def unload_lora(self, slot: int):
        """Empty slot `slot`: requests may no longer name it."""
        if self.lora is None:
            raise ValueError("unload_lora: the engine has no adapter slots (EngineConfig.max_loras is 0)")
        self.lora.unload(slot)

    def _lora_slots(self, lora_ids_list, batch_size: int, ignore_kvcache: bool) -> Optional[list]:
        """The validated per-entry slots, or None when no entry is adapted (the step is then exactly the unadapted one)."""
        if lora_ids_list is None:
            return None
        if ignore_kvcache:
            raise ValueError("lora_ids_list does not apply to the profiling forward (ignore_kvcache)")
        if len(lora_ids_list) != batch_size:
            raise ValueError(f"lora_ids_list has {len(lora_ids_list)} entries for {batch_size} batch entries")
        slots = []
        for i, s in enumerate(lora_ids_list):
            if s is not None:
                if isinstance(s, bool) or not isinstance(s, (int, np.integer)):
                    raise ValueError(f"lora_ids_list[{i}] must be None or a slot id, got {s!r}")
                s = int(s)
                if self.lora is None or not 0 <= s < self.lora.max_loras or not self.lora.loaded[s]:
                    raise ValueError(f"lora_ids_list[{i}]: adapter slot {s} is not loaded")
            slots.append(s)
        return slots if any(s is not None for s in slots) else None

    def _shard_lm_head(self) -> bool:
        want = getattr(self.engine_config, "shard_lm_head", None)
        if want is None:
            want = self.tp_size >= 2 and self.model_config.vocab_size % self.tp_size == 0
        return bool(want) and self.tp_size > 1

    def _kvslot_bytes(self) -> int:
        return self.model_config.get_kvslot_size(self.dtype) // self.tp_size

    @torch.inference_mode()
    def profile_num_blocks(self) -> int:
        """model.py:94-131: forged maximum-size prefill, peak memory -> number of KV blocks that fit."""
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        num_tokens = self.engine_config.max_tokens_in_batch
        batch_size = self.engine_config.max_batch_size
        input_lens = [num_tokens // batch_size] * batch_size
        input_lens[-1] += num_tokens % batch_size
        input_ids = [[0] * n for n in input_lens]
        self.k_cache = self.v_cache = None
        _ = self.forward(input_ids, list(range(batch_size)), [], ignore_kvcache=True)
        torch.cuda.synchronize()
        free_memory, total_memory = torch.cuda.mem_get_info()
        peak_memory = total_memory - free_memory
        useable_memory = total_memory * self.engine_config.gpu_mem_utilization
        print(f"[Model.profile] GPU total memory: {total_memory/GB:.2f} GB, runtime peak memory: {peak_memory/GB:.2f} GB")
        if useable_memory < peak_memory:
            raise RuntimeError(f"Peak memory {peak_memory/GB:.2f} GB exceeds usable memory {useable_memory/GB:.2f} GB "
                               f"({total_memory/GB:.2f} GB * {self.engine_config.gpu_mem_utilization})")
        block_size_bytes = self.engine_config.block_size * self._kvslot_bytes()
        num_gpu_blocks = math.floor((useable_memory - peak_memory) / block_size_bytes)
        torch.cuda.empty_cache()
        if self.tp_size > 1:
            # every rank must run the SAME allocator state (block ids and the out-of-blocks RuntimeError are decided on each
            # rank's host mirror): take the minimum over ranks
            t = torch.tensor([num_gpu_blocks], dtype=torch.int64, device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.tp_group)
            num_gpu_blocks = int(t.item())
        return num_gpu_blocks

    @torch.inference_mode()
    def init_kvcache_and_swap(self, num_blocks: int):
        """model.py:134-175.  KV cache [num_blocks, L, nkv/tp, block_size, D] (zeros, like the reference), CPU swap
        space (pinned here), and the two block managers."""
        if self.tp_size > 1 and dist.is_initialized():
            # identical num_blocks on every rank <=> identical block ids and a collective out-of-blocks decision (all ranks
            # raise the same RuntimeError at the same step instead of one rank leaving its peers inside an exchange)
            t = torch.tensor([num_blocks, -num_blocks], dtype=torch.int64, device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.tp_group)
            if int(t[0].item()) != num_blocks or int(-t[1].item()) != num_blocks:
                raise RuntimeError(f"init_kvcache_and_swap: num_blocks differs between tensor-parallel ranks "
                                   f"(this rank {num_blocks}, min {int(-t[1].item())}, max {int(t[0].item())}); use the value "
                                   f"profile_num_blocks() returns (it is min-reduced over ranks)")
        self.num_blocks = num_blocks
        mc, ec = self.model_config, self.engine_config
        shape = (num_blocks, mc.num_layers, mc.num_kv_heads // self.tp_size, ec.block_size, mc.head_dim)
        self.k_cache = torch.zeros(shape, dtype=self.dtype, device=self.device)
        self.v_cache = torch.zeros(shape, dtype=self.dtype, device=self.device)
        sshape = (ec.num_cpu_blocks,) + shape[1:]
        pin = bool(getattr(ec, "pin_swap_space", True)) and ec.num_cpu_blocks > 0
        self.k_swap = torch.zeros(sshape, dtype=self.dtype, device="cpu", pin_memory=pin)
        self.v_swap = torch.zeros(sshape, dtype=self.dtype, device="cpu", pin_memory=pin)
        # 4 B per token; left uninitialised (no device work): a position is always written before a penalised step reads it
        self.token_cache = torch.empty((num_blocks, ec.block_size), dtype=torch.int32, device=self.device)
        self.token_swap = torch.empty((ec.num_cpu_blocks, ec.block_size), dtype=torch.int32, device="cpu", pin_memory=pin)
        self._penalties_used = False
        self.gpu_block_manager = BlockManager("GPU", num_blocks, ec.max_seqs_in_block_table, ec.max_blocks_per_seq,
                                              ec.block_size, device=self.device)
        self.cpu_block_manager = BlockManager("CPU", ec.num_cpu_blocks, ec.max_seqs_in_block_table,
                                              ec.max_blocks_per_seq, ec.block_size, device=self.device)
        self._graphs = {}

    # ------------------------------------------------------------------ forward
    @torch.inference_mode()
    def _forward(self, input_ids: torch.Tensor, infer_state: LlamaInferState, k_cache=None, v_cache=None,
                 block_table=None) -> torch.Tensor:
        """model.py:228-249."""
        input_embds = self.pre_layer.forward(input_ids)
        self._wait_for_swaps()          # first KV-cache access of the step is layer 0's store: pending swap copies must be done
        residual_buf = torch.zeros_like(input_embds)
        k_cache = self.k_cache if k_cache is None else k_cache
        v_cache = self.v_cache if v_cache is None else v_cache
        if block_table is None and not infer_state.ignore_kvcache:
            block_table = self.gpu_block_manager.block_table
        for layer in self.transformer_layers:
            input_embds = layer.forward(input_embds, residual_buf, k_cache, v_cache, block_table, infer_state)
        if self.comm is not None and residual_buf.shape[0] <= self.comm.max_fused_tokens:
            # the last layer's down_proj partials are still un-reduced: exchange + add + final RMSNorm in one kernel
            normed = self.comm.reduce_add_norm(1, residual_buf.shape[0], residual_buf, self.weight.final_norm,
                                               self.model_config.rms_norm_eps)
            return self.post_layer.forward(normed, infer_state, already_normed=True)
        input_embds += residual_buf
        return self.post_layer.forward(input_embds, infer_state)

    _STAGE_SLOTS = 4

    def _stage_slot(self, n: int):
        """Next slot of the persistent pinned ring, grown geometrically; waits (host side) for the copy that last used it."""
        i = self._stage_next
        self._stage_next = (i + 1) % self._STAGE_SLOTS
        if len(self._stage_ring) <= i:
            self._stage_ring.append(None)
        slot = self._stage_ring[i]
        if slot is None or slot[0].numel() < n:
            cap = max(4096, 1 << (max(n, 1) - 1).bit_length())
            if slot is not None:
                slot[1].synchronize()
            slot = (torch.empty((cap,), dtype=torch.int32).pin_memory(), torch.cuda.Event())
            self._stage_ring[i] = slot
        else:
            slot[1].synchronize()                # no-op unless the copy engine is more than _STAGE_SLOTS steps behind
        return slot

    def _wait_for_swaps(self):
        """Device-side wait (no host sync) for swap copies enqueued on the copy stream since the last forward."""
        if self._swap_done is not None and not (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()):
            torch.cuda.current_stream().wait_event(self._swap_done)
            self._swap_done = None

    def _stage_metadata(self, *parts, out: Optional[torch.Tensor] = None):
        """One persistent pinned host buffer (ring of slots), one async H2D copy; returns int32 device views (one per list), or
        with `out` (a graph's static buffer of exactly that size) copies into it and returns None."""
        n = sum(len(p) for p in parts)
        host, ev = self._stage_slot(n)
        hv, off = host.numpy(), 0
        for p in parts:
            hv[off:off + len(p)] = p
            off += len(p)
        if out is not None:
            out.copy_(host[:n], non_blocking=True)
            ev.record()
            return None
        dev = host[:n].to(self.device, non_blocking=True)
        ev.record()
        views, off = [], 0
        for p in parts:
            views.append(dev[off:off + len(p)])
            off += len(p)
        return views

    def _infer_state(self, ids, seq_ids, seq_lens, p_lens, p_starts, pos, last, *, max_prefill_len: int, max_decoding_len: int,
                     decoding_lens: Optional[list], prefix=None, max_prefill_kv_len: int = 0, speculative: bool = False,
                     ignore_kvcache: bool = False, words=None, filtered: bool = False, sampled: bool = True, sampling_pos=None,
                     top_n: Optional[int] = None, prompt_state: Optional[PromptLogprobsState] = None, block_table=None,
                     token_cache=None, constraints=None, lora_tiles_view=None, truncated: bool = False) -> LlamaInferState:
        """The LlamaInferState of a step from its int32 device views (input ids, block-table rows, sequence lengths with the
        prefill entries first, prompt lengths and first rows, positions, rows to sample) and the sizes the host knows; the batch
        counts are the views' shapes.  decoding_lens: host decode lengths for the reference's split heuristic, None in a graph
        captured for a length bucket (the largest split).  prefix: first position of each chunk (chunked prefill, speculative
        verification), with max_prefill_kv_len.  words: staged sampling_params.sampling_words, noise counter `sampling_pos`
        (default: the sequence lengths), ending with the min-p / typical-p / XTC words when `truncated`; with penalties the sampling state also carries the token history: the input ids, the
        block table and the token pages (default: the model's).  constraints: (device view of the staged constraint region, its
        sampling_params.ConstraintWords) or None.  lora_tiles_view: the staged LoRA tile words or None."""
        mc = self.model_config
        B, T, P = seq_ids.shape[0], ids.shape[0], p_lens.shape[0]
        num_prefill_tokens = T - (B - P)
        sampling = None
        if words is not None:
            sampling = SamplingState.from_staged(words, seq_lens if sampling_pos is None else sampling_pos, filtered, sampled,
                                                 truncated)
            if sampling.penalized:
                sampling = dataclasses.replace(
                    sampling, input_ids=ids, block_table=self.gpu_block_manager.block_table if block_table is None else block_table,
                    token_cache=self.token_cache if token_cache is None else token_cache)
        sbs = 2048 if decoding_lens is None else select_seq_block_size(mc.num_kv_heads, decoding_lens, max_decoding_len)
        return LlamaInferState(
            batch_size=B, num_tokens=T, seq_ids=seq_ids, softmax_scale=mc.head_dim ** -0.5,
            num_prefill_seqs=P, num_prefill_tokens=num_prefill_tokens, prefill_seq_start_locs=p_starts,
            # ends at num_prefill_tokens (the reference puts num_tokens there, model.py:336-339, which over-declares
            # the last prompt by the number of decoding tokens on mixed batches; SURVEY.md §3.1)
            prefill_seq_start_locs_with_end=torch.cat([p_starts, p_starts.new_tensor([num_prefill_tokens])]) if P > 0 else p_starts,
            prefill_seq_lens=p_lens, max_prefill_len=max_prefill_len,
            num_decoding_seqs=B - P, decoding_seq_lens=seq_lens[P:], max_decoding_len=max_decoding_len,
            seq_block_size=sbs, num_seq_blocks=(max_decoding_len + sbs - 1) // sbs,
            position_cos=self._cos_cached.index_select(0, pos), position_sin=self._sin_cached.index_select(0, pos),
            ignore_kvcache=ignore_kvcache, paged_attn_seq_block_size=0, last_token_indices=last,
            prefill_prefix_lens=prefix, max_prefill_kv_len=max_prefill_kv_len, speculative=speculative,
            sampling=sampling, logprobs=top_n, prompt_logprobs=prompt_state,
            constraints=None if constraints is None else ConstraintState.from_staged(constraints[0], *constraints[1][1:]),
            lora=None if lora_tiles_view is None else LoraState(self.lora, lora_tiles_view.view(-1, 3)))

    @torch.inference_mode()
    def forward(self, input_ids_list: list, seq_ids_list: list, decoding_seq_lens_list: list,
                ignore_kvcache: bool = False, prefill_prefix_lens_list: Optional[list] = None,
                sampling_params_list: Optional[list] = None, token_masks_list: Optional[list] = None,
                lora_ids_list: Optional[list] = None) -> list:
        """model.py:252-359.  Batch layout contract: prefill sequences first (full prompt each), then decoding
        sequences (exactly one token each); decoding_seq_lens_list[i] includes the new token.

        `prefill_prefix_lens_list` (addition, SURVEY.md §8 f-1: chunked / SARATHI-style prefill, which the reference's
        forward cannot express): when given, prefill entry i is the CHUNK of its prompt that starts at position
        prefill_prefix_lens_list[i]; positions below it were written to the KV cache by earlier calls.  The chunk's
        K/V are stored at their positions and its queries attend to the whole prefix + chunk through the block
        table.  The token returned for a prefill entry is sampled after the chunk's last token (meaningful for the
        final chunk of a prompt only).

        `sampling_params_list` (addition): one swiftllm_b200.SamplingParams per batch entry; the token of entry i is drawn with
        its temperature / top-k / top-p and seed (csrc/sampling.cu), the noise keyed by the sequence length after this step.
        None (or every temperature 0) is greedy decoding, the reference's behaviour.  Entries with repetition / frequency /
        presence penalties have their logits penalised first (csrc/penalties.cu), over the history recorded in the token pages:
        such a request must carry the same parameters from its first prefill chunk on.  The no-repeat n-gram ban and DRY
        (SamplingParams.no_repeat_ngram_size, dry_*) read the same history in the same launch, after the penalties, with the
        same contract.  Invalid parameters (and penalties or n-gram controls with ignore_kvcache, which has no block table to
        record into, or a DRY breaker id outside [0, vocab_size)) raise ValueError before anything is enqueued.

        `token_masks_list` (addition, constrained decoding): None, or one entry per batch entry - None (unconstrained) or a packed
        allowed-token mask, a numpy array or CPU tensor of int32 / uint32 with W = ceil(vocab_size / 32) words, bit v % 32 of word
        v // 32 set = id v allowed (the layout of xgrammar and vLLM; swiftllm_b200.token_mask builds one; bits past vocab_size are
        ignored).  Disallowed ids become -inf, then SamplingParams.logit_bias is added, both before the penalties
        (csrc/constraints.cu).  A mask of the wrong shape or dtype, one that allows no id, a list of the wrong length, a bias id
        outside [0, vocab_size) and masks with ignore_kvcache raise ValueError before anything is enqueued.

        `lora_ids_list` (addition, multi-LoRA): None, or one entry per batch entry - None (the base model) or a slot loaded with
        load_lora; the entry's rows run with that adapter at every projection (csrc/lora.cu).  K/V cached by an adapted entry
        depend on its adapter: keep a sequence on one slot (and fork it only to sequences of the same slot).  A list of the wrong
        length, a slot that is not loaded and use with ignore_kvcache raise ValueError before anything is enqueued.  A list of
        None entries is a step without adapters."""
        return self.forward_async(input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache,
                                  prefill_prefix_lens_list, sampling_params_list, token_masks_list, lora_ids_list).tolist()

    @torch.inference_mode()
    def forward_async(self, input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache=False,
                      prefill_prefix_lens_list=None, sampling_params_list=None, token_masks_list=None,
                      lora_ids_list=None) -> torch.Tensor:
        """Same as forward() but returns the token tensor on the device (no sync)."""
        return self._step(input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache, prefill_prefix_lens_list,
                          sampling_params_list, with_logprobs=False, token_masks_list=token_masks_list,
                          lora_ids_list=lora_ids_list)

    @torch.inference_mode()
    def forward_with_logprobs(self, input_ids_list: list, seq_ids_list: list, decoding_seq_lens_list: list,
                              ignore_kvcache: bool = False, prefill_prefix_lens_list: Optional[list] = None,
                              sampling_params_list: Optional[list] = None, prompt_next_ids_list: Optional[list] = None,
                              token_masks_list: Optional[list] = None, lora_ids_list: Optional[list] = None) -> list:
        """forward() that also returns log-probabilities: one swiftllm_b200.TokenLogprobs(token, logprob, top, prompt) per batch
        entry.  Entry i gets them when sampling_params_list[i].logprobs is not None: the log-probability of its token and, for
        logprobs = N > 0, the N most likely tokens as (id, logprob), most likely first, ties broken by the smaller id.  They are
        log_softmax of the raw logits the token was chosen from (csrc/logprobs.cu), not of the temperature-scaled or filtered
        distribution.  The tokens are the ones forward() returns for the same arguments (token_masks_list included: the
        log-probabilities stay those of the unconstrained logits).

        A prefill entry with sampling_params_list[i].prompt_logprobs set also gets `prompt`, a swiftllm_b200.PromptLogprobs: each
        of its rows scores the prompt token after it (csrc/prompt_logprobs.cu, the same values as above).  The last row of the
        entry scores prompt_next_ids_list[i] when that is given (one entry per prefill entry, None or the id of the prompt token
        after this chunk); so chunks of a prompt, each given the next chunk's first token, together score positions 1 .. P - 1.
        The step's tokens and KV-cache writes are those of forward().  A prompt_next_ids_list of the wrong length, or an id of an
        asking entry outside [0, vocab_size), raises ValueError before anything is enqueued.  With lora_ids_list, every
        log-probability (prompt ones included) is the adapted model's."""
        plan = self._prompt_plan(input_ids_list, decoding_seq_lens_list, prefill_prefix_lens_list, sampling_params_list,
                                 prompt_next_ids_list)
        out = self._step(input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache, prefill_prefix_lens_list,
                         sampling_params_list, with_logprobs=True, prompt_plan=plan if plan and plan["num_rows"] else None,
                         token_masks_list=token_masks_list, lora_ids_list=lora_ids_list)
        prompt_out = None
        if plan and plan["num_rows"]:
            out, prompt_out = out
        if isinstance(out, torch.Tensor):                   # no entry asked for the returned token's log-probabilities
            res = [TokenLogprobs(t) for t in out.tolist()]
        else:
            tokens, token_lp, top_ids, top_lp = (t.tolist() for t in out)
            res = []
            for i, t in enumerate(tokens):
                n = sampling_params_list[i].logprobs
                if n is None:
                    res.append(TokenLogprobs(t))
                else:
                    n = min(int(n), self.model_config.vocab_size)
                    res.append(TokenLogprobs(t, token_lp[i], list(zip(top_ids[i][:n], top_lp[i][:n]))))
        if plan:
            lp, rank, ids, tlp = (t.cpu().numpy() for t in prompt_out) if prompt_out is not None else (None,) * 4
            for i, first, off, k, n in plan["entries"]:
                tgt = np.asarray(plan["targets"][off:off + k], dtype=np.int64)
                if k == 0:
                    pl = PromptLogprobs(first, tgt, np.zeros((0,), np.float32), np.zeros((0,), np.int32),
                                        np.zeros((0, n), np.int32), np.zeros((0, n), np.float32))
                else:
                    pl = PromptLogprobs(first, tgt, lp[off:off + k].copy(), rank[off:off + k].copy(),
                                        ids[off:off + k, :n].copy(), tlp[off:off + k, :n].copy())
                res[i] = res[i]._replace(prompt=pl)
        return res

    def _prompt_plan(self, input_ids_list, decoding_seq_lens_list, prefill_prefix_lens_list, sampling_params_list,
                     prompt_next_ids_list):
        """Host plan of the prompt rows of forward_with_logprobs, None when no prefill entry asks: entries [(batch index, first
        position, offset into the rows, rows k, N)], pieces [(first row of the entry in the activation matrix, its token
        count n, next id or None)] of the entries with rows to score, the number of rows, the targets and the per-launch N.
        Validates prompt_next_ids_list (ValueError)."""
        P = len(input_ids_list) - len(decoding_seq_lens_list)
        if prompt_next_ids_list is not None and len(prompt_next_ids_list) != P:
            raise ValueError(f"prompt_next_ids_list has {len(prompt_next_ids_list)} entries for {P} prefill entries")
        if sampling_params_list is None or len(sampling_params_list) != len(input_ids_list):
            return None                                     # sampling_words raises for a list of the wrong length
        for sp in sampling_params_list[:P]:
            if not isinstance(sp, SamplingParams):
                return None                                 # sampling_words raises
            sp.validate()
        top_n = prompt_logprobs_top_n(sampling_params_list[:P])
        if top_n is None:
            return None
        V = self.model_config.vocab_size
        prefix = [int(x) for x in prefill_prefix_lens_list] if prefill_prefix_lens_list is not None else [0] * P
        entries, pieces, targets = [], [], []
        start = 0
        for i in range(P):
            ids, n_i = input_ids_list[i], len(input_ids_list[i])
            n = sampling_params_list[i].prompt_logprobs
            if n is not None:
                nxt = None if prompt_next_ids_list is None else prompt_next_ids_list[i]
                if nxt is not None and (isinstance(nxt, bool) or not isinstance(nxt, (int, np.integer)) or not 0 <= nxt < V):
                    raise ValueError(f"prompt_next_ids_list[{i}] must be None or a token id in [0, {V}), got {nxt!r}")
                k = max(n_i - 1, 0) + (nxt is not None and n_i > 0)
                entries.append((i, prefix[i] + 1, len(targets), k, min(int(n), V)))
                targets += [int(x) for x in ids[1:]]
                if nxt is not None and n_i > 0:
                    targets.append(int(nxt))
                if k > 0:
                    pieces.append((start, n_i, None if nxt is None else int(nxt)))
            start += n_i
        return dict(entries=entries, pieces=pieces, num_rows=len(targets), targets=targets, top_n=top_n)

    def _prompt_block_rows(self) -> int:
        """Rows per prompt-logprobs block: the block's logits (and with a sharded lm_head the shard and the gathered copy) stay
        within the [max_tokens_in_batch, 2 * ffn_inter_dim / tp] up_gate output of the forward profile_num_blocks measures."""
        mc = self.model_config
        V = mc.vocab_size
        per_row = 2 * V + V // self.tp_size if self.post_layer.sharded else V
        return max(1, self.engine_config.max_tokens_in_batch * 2 * (mc.ffn_inter_dim // self.tp_size) // per_row)

    MAX_SPECULATIVE_ROWS = 8

    @torch.inference_mode()
    def forward_speculative(self, input_ids_list: list, seq_ids_list: list, prefix_lens_list: list,
                            sampling_params_list: Optional[list] = None, ignore_kvcache: bool = False,
                            token_masks_list: Optional[list] = None, lora_ids_list: Optional[list] = None) -> list:
        """Speculative decoding: score a plain decode input and up to 7 caller-made drafts per sequence in one step.

        Entry i is input_ids_list[i] = [x, d_1, ..., d_k] (1 <= k + 1 <= 8): x is the token a plain decode step would feed, d_* are
        drafts (prompt lookup, an n-gram table, another model's greedy output).  prefix_lens_list[i] tokens of the sequence are in
        the KV cache (decoding_seq_len - 1 of the equivalent forward() step); row j sits at position prefix_i + j.  For every row
        j, y_j is the token forward() would return for a decode step at that position: argmax, or the sampling kernel with the
        entry's SamplingParams (one seed for all the entry's rows) and pos = prefix_i + j + 1.  With n the number of leading
        drafts such that d_{j+1} == y_j, entry i returns [y_0, ..., y_n]: exactly the tokens n + 1 plain steps would return.

        Afterwards the sequence has prefix_i + 1 + n cached tokens and holds ceil((prefix_i + 1 + n) / block_size) blocks: continue
        it with forward() at decoding_seq_len prefix_i + n + 2 and input y_n, or with forward_speculative at prefix prefix_i + 1 + n.
        K/V of rejected rows inside a kept block are overwritten by later steps (attention never reads past a row's position).
        Speculative entries only (no prompts in the same call); runs eagerly and syncs once, like forward().  Raises ValueError
        before anything is enqueued for: a row count outside [1, 8], a negative prefix or one whose rows run past the position
        table, ignore_kvcache, invalid sampling parameters, penalties and n-gram controls.  SamplingParams.logprobs is ignored.

        token_masks_list: None, or per entry None or a [k + 1, W] mask array (forward()'s layout, one row per input row): row j holds
        the constraint state after x, d_1 .. d_j, the mask the caller would pass to the plain step at that position; the entry's
        logit_bias applies to all its rows.  A draft its row's mask disallows can never equal y_j, so acceptance stops there.  A
        mask with the wrong row count raises ValueError like forward()'s checks.  lora_ids_list: forward()'s, one slot per
        entry, shared by all its rows."""
        B = len(input_ids_list)
        if len(seq_ids_list) != B or len(prefix_lens_list) != B:
            raise ValueError(f"forward_speculative: {B} entries but {len(seq_ids_list)} seq ids and {len(prefix_lens_list)} prefixes")
        if ignore_kvcache:
            raise ValueError("forward_speculative reads and writes the KV cache: ignore_kvcache is not applicable")
        rows = [len(x) for x in input_ids_list]
        prefix = [int(p) for p in prefix_lens_list]
        max_pos = self._cos_cached.shape[0]
        for n, p in zip(rows, prefix):
            if not 1 <= n <= self.MAX_SPECULATIVE_ROWS:
                raise ValueError(f"forward_speculative: an entry has {n} rows; 1 to {self.MAX_SPECULATIVE_ROWS} are supported")
            if p < 0 or p + n > max_pos:
                raise ValueError(f"forward_speculative: prefix {p} with {n} rows is outside the position table [0, {max_pos})")
        samp = None if sampling_params_list is None else sampling_words(sampling_params_list, B, self._sampling_rng)
        if has_penalties(sampling_params_list):
            raise ValueError("forward_speculative does not apply penalties (their history is per position)")
        if has_ngram_controls(sampling_params_list):
            raise ValueError("forward_speculative does not apply no_repeat_ngram_size or DRY (their history is per position)")
        truncated = has_truncation(sampling_params_list)
        con = constraint_words(token_masks_list, sampling_params_list, B, self.model_config.vocab_size, rows=rows)
        slots = self._lora_slots(lora_ids_list, B, False)
        if B == 0:
            return []
        self._check_shared_writes(seq_ids_list, prefix)
        T = sum(rows)
        rep = np.repeat(np.arange(B), rows)
        flat_ids = list(itertools.chain(*input_ids_list))
        starts = list(itertools.accumulate([0] + rows[:-1]))
        positions = [p + j for p, n in zip(prefix, rows) for j in range(n)]
        seq_lengths = [p + n for p, n in zip(prefix, rows)]
        row_pos = [q + 1 for q in positions]             # sampling noise counter of row j: prefix + j + 1
        if samp is not None:
            # the words are per entry: every row of an entry gets its parameters and its seed
            # (the min-p / typical-p / XTC words, when staged, follow the 5 * B sampling words: penalties are refused above)
            w = np.asarray(samp[0], dtype=np.int64)
            row_words = np.concatenate([w[:2 * B].reshape(B, 2)[rep].reshape(-1)] +
                                       [w[(2 + s) * B:(3 + s) * B][rep] for s in range(3 + 4 * truncated)]).tolist()
        tiles = None if slots is None else lora_tiles(slots, rows)
        if tiles is not None:
            self.lora.ensure_rows(T)
        views = self._stage_metadata(*([row_words] if samp else []), *([con.words] if con else []),
                                     *([tiles] if tiles else []), flat_ids, seq_ids_list, seq_lengths, rows, starts, positions,
                                     range(T), prefix, row_pos)
        ids, seq_ids, seq_lens, p_lens, p_starts, pos, last, p_prefix, r_pos = views[-9:]
        bm = self.gpu_block_manager
        bm.allocate_blocks_for_seqs(seq_ids, seq_lens, seq_ids_list=seq_ids_list, target_lens_list=seq_lengths,
                                    want_new_blocks=False)
        infer_state = self._infer_state(ids, seq_ids, seq_lens, p_lens, p_starts, pos, last, max_prefill_len=max(rows),
                                        max_decoding_len=0, decoding_lens=[], prefix=p_prefix,
                                        max_prefill_kv_len=max(seq_lengths), speculative=True,
                                        words=views[0] if samp else None, filtered=bool(samp and samp[1]), sampling_pos=r_pos,
                                        truncated=truncated, constraints=None if con is None else (views[1 if samp else 0], con),
                                        lora_tiles_view=views[bool(samp) + bool(con)] if tiles else None)
        tokens = self._forward(ids, infer_state).tolist()
        out, keep = [], []
        for ids_i, s, n_rows, p in zip(input_ids_list, starts, rows, prefix):
            y = tokens[s:s + n_rows]
            n = 0
            while n < n_rows - 1 and int(ids_i[n + 1]) == y[n]:
                n += 1
            out.append(y[:n + 1])
            keep.append(p + 1 + n)
        # give back the blocks that only held rejected rows
        bs = bm.block_size
        if any((k + bs - 1) // bs < (L + bs - 1) // bs for k, L in zip(keep, seq_lengths)):
            bm.truncate_blocks_for_seqs(seq_ids, torch.tensor(keep, dtype=torch.int32, device=self.device),
                                        seq_ids_list=seq_ids_list, target_lens_list=keep)
        return out

    def _step(self, input_ids_list, seq_ids_list, decoding_seq_lens_list, ignore_kvcache, prefill_prefix_lens_list,
              sampling_params_list, with_logprobs: bool, prompt_plan: Optional[dict] = None, token_masks_list=None,
              lora_ids_list=None):
        """One step: the token tensor, or with log-probabilities asked for by some entry (with_logprobs and a
        SamplingParams.logprobs set) the tuple (tokens, token logprobs, top ids, top logprobs) on the device.  With a
        `prompt_plan` (forward_with_logprobs._prompt_plan, some rows to score): (that, (prompt logprobs, ranks, top ids, top
        logprobs)).  The step stages exactly what it stages without one: the post layer builds the rows and targets on the device
        after the layers, so nothing of the prompt part is allocated while the forward's activations are.  token_masks_list and
        logit_bias add the constraint region (sampling_params.constraint_words) after the sampling words; without them the step
        stages, launches and keys its graph exactly as before; so does lora_ids_list with the LoRA tile list (after those)."""
        samp = None if sampling_params_list is None else \
            sampling_words(sampling_params_list, len(input_ids_list), self._sampling_rng)
        top_n = logprobs_top_n(sampling_params_list) if with_logprobs else None
        ngram = has_ngram_controls(sampling_params_list)
        penalized = ngram or has_penalties(sampling_params_list)
        truncated = has_truncation(sampling_params_list)
        if ngram and ignore_kvcache:
            raise ValueError("no_repeat_ngram_size and DRY need the token history of the block table: not available with "
                             "ignore_kvcache")
        if penalized and ignore_kvcache:
            raise ValueError("penalties need the token history of the block table: not available with ignore_kvcache")
        if ngram:
            check_breaker_ids(sampling_params_list, self.model_config.vocab_size)
        if token_masks_list is not None and ignore_kvcache:
            raise ValueError("token_masks_list does not apply to the profiling forward (ignore_kvcache)")
        slots = self._lora_slots(lora_ids_list, len(input_ids_list), ignore_kvcache)
        sampled = samp is not None and any(sp.temperature > 0 for sp in sampling_params_list)
        num_prefill_seqs = len(input_ids_list) - len(decoding_seq_lens_list)
        flat_ids = list(itertools.chain(*input_ids_list))
        prefill_lens = [len(s) for s in input_ids_list[:num_prefill_seqs]]
        chunked = prefill_prefix_lens_list is not None and num_prefill_seqs > 0
        if chunked:
            prefix_lens = [int(x) for x in prefill_prefix_lens_list]
            assert len(prefix_lens) == num_prefill_seqs and min(prefix_lens) >= 0, \
                "prefill_prefix_lens_list needs one non-negative entry per prefill sequence"
            assert not ignore_kvcache, "chunked prefill reads the KV cache: ignore_kvcache is not applicable"
            # first chunks only (every prefix 0): nothing to read back from the cache, so this IS the reference's whole-prompt
            # contract - packed-k/v attention and the plain store
            chunked = max(prefix_lens) > 0
        else:
            prefix_lens = [0] * num_prefill_seqs
        seq_lengths_list = [p + n for p, n in zip(prefix_lens, prefill_lens)] + list(decoding_seq_lens_list)
        batch_size, num_tokens = len(input_ids_list), len(flat_ids)
        num_prefill_tokens = num_tokens - (batch_size - num_prefill_seqs)
        prefill_starts = list(itertools.accumulate([0] + prefill_lens[:-1])) if prefill_lens else []
        max_prefill_len = max(prefill_lens) if prefill_lens else 0
        max_decoding_len = max(decoding_seq_lens_list) if decoding_seq_lens_list else 0
        positions = [p0 + p for p0, n in zip(prefix_lens, prefill_lens) for p in range(n)] + \
            [l - 1 for l in decoding_seq_lens_list]
        last_idx = [s + n - 1 for s, n in zip(prefill_starts, prefill_lens)] + list(range(num_prefill_tokens, num_tokens))

        graph = (getattr(self.engine_config, "use_cuda_graph", False) and num_prefill_seqs == 0 and not ignore_kvcache
                 and batch_size > 0)
        con = constraint_words(token_masks_list, sampling_params_list, batch_size, self.model_config.vocab_size, graph=graph)
        if slots is not None:
            self.lora.ensure_rows(num_tokens)
        if graph:
            return self._forward_decode_graph(flat_ids, seq_ids_list, list(decoding_seq_lens_list), max_decoding_len, samp,
                                              top_n, penalized, sampled, con, slots, ngram, truncated)
        tiles = None if slots is None else lora_tiles(slots, prefill_lens + [1] * (batch_size - num_prefill_seqs))

        if not ignore_kvcache:
            self._check_shared_writes(seq_ids_list, prefix_lens + [l - 1 for l in decoding_seq_lens_list])
        # the sampling words go first: the int64 seeds need an 8-byte aligned offset
        views = self._stage_metadata(
            *([samp[0]] if samp else []), *([con.words] if con else []), *([tiles] if tiles else []), flat_ids, seq_ids_list,
            seq_lengths_list, prefill_lens, prefill_starts, positions, last_idx, prefix_lens if chunked else [])
        ids, seq_ids, seq_lengths, p_lens, p_starts, pos, last, p_prefix = views[-8:]
        pp = prompt_plan
        prompt_state = None if pp is None else PromptLogprobsState(
            pieces=pp["pieces"], num_rows=pp["num_rows"], input_ids=ids, top_n=pp["top_n"], block_rows=self._prompt_block_rows())
        self._penalties_used |= penalized

        if not ignore_kvcache:
            self.gpu_block_manager.allocate_blocks_for_seqs(seq_ids, seq_lengths, seq_ids_list=seq_ids_list,
                                                            target_lens_list=seq_lengths_list, want_new_blocks=False)

        infer_state = self._infer_state(
            ids, seq_ids, seq_lengths, p_lens, p_starts, pos, last, max_prefill_len=max_prefill_len,
            max_decoding_len=max_decoding_len, decoding_lens=list(decoding_seq_lens_list), prefix=p_prefix if chunked else None,
            max_prefill_kv_len=max(seq_lengths_list[:num_prefill_seqs]) if chunked else 0, ignore_kvcache=ignore_kvcache,
            words=views[0] if samp else None, filtered=bool(samp and samp[1]), sampled=sampled, top_n=top_n,
            truncated=truncated, prompt_state=prompt_state, constraints=None if con is None else (views[1 if samp else 0], con),
            lora_tiles_view=views[bool(samp) + bool(con)] if tiles else None)
        return self._forward(ids, infer_state)

    # ------------------------------------------------------------------ CUDA-graph decode path
    def _forward_decode_graph(self, flat_ids, seq_ids_list, lens_list, max_len, samp=None, top_n=None, penalized=False,
                              sampled=True, con: Optional[ConstraintWords] = None, slots: Optional[list] = None,
                              ngram: bool = False, truncated: bool = False):
        """Pure-decode step replayed from a CUDA graph.  The step's metadata is staged through the same pinned ring as an eager
        step's, into the graph's static device buffer, and its blocks are reserved on the manager's host mirror like an eager
        step's; the graph (keyed by batch size and the attention launch geometry) contains allocation-free work only: block
        allocation, gathers, every layer, lm_head and argmax - or, for sampled steps (`samp`: staged sampling words and the
        filtered flag, sampling_params.sampling_words), the sampling kernel, with the parameters staged in the same copy.  A step
        with log-probabilities (`top_n`) has its own graph, which also runs the log-probability kernel; so has a step with
        penalties, which also runs the penalty kernel (and the argmax instead of the sampling kernel when no row samples), and a
        step with n-gram controls (`ngram`) the penalty kernel's n-gram launch, keyed by one more tag.  A
        constrained step (`con`: the graph-sized constraint region) has its own graph per bias capacity (the step's bias entries
        rounded up to a power of two), which also runs the constraint kernel.  An adapted step (`slots`, _lora_slots) has its own
        graph, which also runs the LoRA kernels over a tile list padded to B tiles, so any mix of slots replays it.  A step
        with min-p / typical-p / XTC rows (`truncated`) has its own graph, which samples through the truncated entry."""
        from swiftllm_b200 import _lib
        self._check_shared_writes(seq_ids_list, [l - 1 for l in lens_list])
        B = len(flat_ids)
        mc = self.model_config
        nkv = mc.num_kv_heads // self.tp_size
        nq = mc.num_q_heads // self.tp_size
        # launch geometry of paged attention depends on max_len only through the split count: bucket it
        bucket = ((max_len + 1023) // 1024) * 1024
        ws_bytes = _lib.lib().sllm_paged_attention_workspace_bytes(B, nq, mc.head_dim, bucket, 0, nkv)
        key = (B, bucket if ws_bytes > 0 else 0)
        if samp:
            # sharded lm_head: filtered rows sample the gathered full rows, the others exchange per-shard pairs
            key += (True, samp[1] and self.post_layer.sharded)
        if top_n is not None:
            key += ("logprobs", top_n)
        if penalized:
            key += ("penalties", sampled) + (("ngram",) if ngram else ())
        if con is not None:
            key += ("constrained", con.num_bias)
        if slots is not None:
            key += ("lora",)
        if truncated:
            key += ("truncated",)
        g = self._graphs.pop(key, None)
        if g is None:
            # bounded cache (least recently used graph dropped first); all graphs share ONE memory pool - they are replayed
            # one at a time on one stream and their only output (`tokens`) is copied out before the next replay
            cap = max(1, int(getattr(self.engine_config, "max_cuda_graphs", 16)))
            while len(self._graphs) >= cap:
                self._graphs.pop(next(iter(self._graphs)))
            g = self._capture_decode_graph(B, bucket, None if not samp else samp[1], top_n, penalized, sampled,
                                           None if con is None else con._replace(words=None),
                                           **({} if slots is None else dict(lora=True)), **(dict(ngram=True) if ngram else {}),
                                           **(dict(truncated=True) if truncated else {}))
        self._graphs[key] = g                    # (re)insert as most recently used
        # the blocks are counted on the host, and the eager step's errors raised, before anything is enqueued; the graph's
        # allocation kernel hands them out
        self.gpu_block_manager.reserve_blocks_for_seqs(seq_ids_list, lens_list)
        tiles = [] if slots is None else lora_tiles(slots, [1] * B, pad_to=B)
        self._stage_metadata(*([samp[0]] if samp else []), *([con.words] if con else []), *([tiles] if tiles else []), flat_ids,
                             seq_ids_list, lens_list, out=g["meta"])
        self._wait_for_swaps()
        self._penalties_used |= penalized
        g["graph"].replay()
        # the graph's static outputs are overwritten by the next replay: hand out copies (stream-ordered, no sync)
        if g["logprobs"] is not None:
            return (g["tokens"].clone(),) + tuple(t.clone() for t in g["logprobs"])
        return g["tokens"].clone()

    def _capture_decode_graph(self, B: int, bucket_len: int, filtered: Optional[bool] = None, top_n: Optional[int] = None,
                              penalized: bool = False, sampled: bool = True, con: Optional[ConstraintWords] = None,
                              lora: bool = False, ngram: bool = False, truncated: bool = False):
        """filtered None: greedy graph; else a sampled graph whose meta starts with the 5 * B sampling words.  top_n: the graph
        also computes log-probabilities with this top-N.  penalized: the meta starts with 8 * B words (sampling and penalties),
        the graph penalises the logits and records the step's tokens in the token pages; `sampled` False takes the argmax.  ngram:
        the meta starts with 28 * B words (the n-gram controls follow the penalties; all zero, so off, during the warm-up).  con:
        the sizes of the graph's constraint region (words None), which follows the sampling words; the graph constrains the
        logits first.  lora: B LoRA tiles follow (empty during the warm-up).  truncated: 4 * B more sampling words (min-p,
        typical-p, XTC) end the sampling words; the warm-up's temperatures are 0, so its rows are greedy."""
        ec = self.engine_config
        dev = self.device
        nw = 0 if filtered is None else (28 if ngram else 8 if penalized else 5) * B + (4 * B if truncated else 0)
        nc = 0 if con is None else ConstraintWords.size(*con[1:])
        nl = 3 * B if lora else 0
        meta = torch.zeros((nw + nc + nl + 3 * B,), dtype=torch.int32, device=dev)
        o = nw + nc + nl
        ids, seq_ids, lens = meta[o:o + B], meta[o + B:o + 2 * B], meta[o + 2 * B:]
        last = torch.arange(B, dtype=torch.int32, device=dev)
        empty = torch.empty((0,), dtype=torch.int32, device=dev)

        def step(bm, k_cache, v_cache, token_cache):
            # the replayed lengths are unknown here: the kernel runs on every replay, reserve_blocks_for_seqs counts its blocks
            bm.allocate_reserved_blocks(seq_ids, lens)
            # `pos` is held until the step returns: the order in which a capture frees its tensors decides where later captures
            # into the shared pool place theirs, and parity tests read post_layer.last_logits, the logits of the graph captured last
            pos = (lens - 1).long()
            st = self._infer_state(ids, seq_ids, lens, empty, empty, pos, last, max_prefill_len=0,
                                   max_decoding_len=bucket_len, decoding_lens=None,
                                   words=None if filtered is None else meta[:nw], filtered=filtered, sampled=sampled,
                                   truncated=truncated,
                                   top_n=top_n, block_table=bm.block_table, token_cache=token_cache,
                                   constraints=None if con is None else (meta[nw:nw + nc], con),
                                   lora_tiles_view=meta[nw + nc:o] if lora else None)
            return self._forward(ids, st, k_cache=k_cache, v_cache=v_cache, block_table=bm.block_table)

        # Warm-up (library handles, lazy kernel loading, GEMM heuristics for these shapes) must not touch the real
        # cache or block tables: it runs against a one-block scratch cache with B one-token sequences.
        scratch_bm = BlockManager("scratch", B, B, 1, ec.block_size, device=dev)
        sshape = (B,) + tuple(self.k_cache.shape[1:])
        k_s = torch.zeros(sshape, dtype=self.dtype, device=dev)
        v_s = torch.zeros(sshape, dtype=self.dtype, device=dev)
        t_s = torch.zeros((B, ec.block_size), dtype=torch.int32, device=dev) if penalized else None
        meta.zero_()
        if con is not None:
            # warm-up region: every row on mask row 0, no bias entries, every id allowed
            meta[nw + nc - con.num_masks * con.mask_words:nw + nc].fill_(-1)
        seq_ids.copy_(torch.arange(B, dtype=torch.int32, device=dev))
        lens.fill_(1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                step(scratch_bm, k_s, v_s, t_s)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        del k_s, v_s, t_s, scratch_bm
        graph = torch.cuda.CUDAGraph()
        if getattr(self, "_graph_pool", None) is None:
            self._graph_pool = torch.cuda.graph_pool_handle()
        with torch.cuda.graph(graph, pool=self._graph_pool):
            out = step(self.gpu_block_manager, self.k_cache, self.v_cache, self.token_cache)
        torch.cuda.synchronize()
        tokens, logprobs = (out, None) if top_n is None else (out[0], out[1:])
        # `last` / `empty` are read by the captured kernels on every replay: keep them alive with the graph, and
        # the LoRA u buffer too: LoraPool.ensure_rows may replace it, and this graph reads the one it was captured with
        return dict(graph=graph, meta=meta, tokens=tokens, logprobs=logprobs,
                    keep=(last, empty) + ((self.lora.u,) if lora else ()))

    # ------------------------------------------------------------------ shared blocks
    def _check_shared_writes(self, seq_ids_list, first_positions):
        """ValueError (before anything is enqueued) when a step would store K/V inside a block its sequence shares with a fork.
        An entry writes the positions from first_positions[i] on, and shared blocks are the leading blocks of a row, so one
        comparison per entry decides it.  Nothing to check until the first fork."""
        bm = self.gpu_block_manager
        if not bm.forked or len(seq_ids_list) == 0:
            return
        shared = bm.get_num_shared_blocks_host(seq_ids_list)
        pos = np.asarray(first_positions, dtype=np.int64)
        bad = pos // bm.block_size < shared
        if bad.any():
            i = int(np.argmax(bad))
            raise ValueError(f"sequence {int(seq_ids_list[i])} would write position {int(pos[i])}, inside one of its first "
                             f"{shared[i]} blocks, which it shares with a fork: shared blocks are read-only")

    @torch.inference_mode()
    def fork_seqs(self, src_seq_ids_list: list, dst_seq_ids_list: list, lens_list: list):
        """Entry i: dst_seq_ids_list[i] holds the first P = lens_list[i] cached tokens of src_seq_ids_list[i], as if they had been
        prefilled into it.  Blocks [0, P // block_size) of src are shared (dst's block-table row points at them, one more owner
        each); when P % block_size != 0, dst gets a fresh block (lowest free id first, batch order) into which src's block
        P // block_size is copied: K and V pages of every layer on this rank and the token page penalties read.  dst then continues
        like any sequence: forward() decode at decoding_seq_len P + 1, chunked prefill with prefill_prefix_lens_list [P], or
        forward_speculative at prefix P.  Several entries may fork the same src (n-way fork), and P may be shorter than what src
        holds.  Sampling is a pure function of (logits, parameters, seed, position): forks decoded with the same fixed seed
        produce identical continuations; parallel sampling uses seed=None or distinct seeds.

        No step may store K/V inside a block that has more than one owner (ValueError before anything is enqueued); a block is
        freed when its last owner is freed or swapped out, and a swapped-out fork comes back with private blocks.  Raises
        ValueError, before anything is enqueued, when the list lengths differ, P < 1 or P > blocks held by src * block_size, src
        holds no GPU blocks (or is swapped out), dst holds blocks on either device, a dst repeats or is also a src, or an id is
        outside [0, max_seqs_in_block_table); RuntimeError when the tail blocks do not fit.  Stream-ordered, no host sync.

        Cached K/V depend on the LoRA adapter that computed them (lora_ids_list): fork only to sequences that continue with the
        source's slot.  The data plane cannot detect a fork across adapters."""
        B = len(src_seq_ids_list)
        if len(dst_seq_ids_list) != B or len(lens_list) != B:
            raise ValueError(f"fork_seqs: {B} sources but {len(dst_seq_ids_list)} destinations and {len(lens_list)} lengths")
        src, dst, lens = ([int(x) for x in l] for l in (src_seq_ids_list, dst_seq_ids_list, lens_list))
        gpu, cpu = self.gpu_block_manager, self.cpu_block_manager
        bs, nseq = gpu.block_size, gpu.block_table.shape[0]
        for sid in src + dst:
            if not 0 <= sid < nseq:
                raise ValueError(f"fork_seqs: sequence id {sid} outside [0, {nseq})")
        if len(set(dst)) != B:
            raise ValueError("fork_seqs: a destination sequence repeats")
        if set(dst) & set(src):
            raise ValueError(f"fork_seqs: sequences {sorted(set(dst) & set(src))} are both a source and a destination")
        on_gpu, on_cpu = gpu.get_num_allocated_blocks_host(src + dst), cpu.get_num_allocated_blocks_host(src + dst)
        for i, (s, d, p) in enumerate(zip(src, dst, lens)):
            if on_cpu[i] > 0:
                raise ValueError(f"fork_seqs: source sequence {s} is swapped out")
            have = on_gpu[i]
            if have == 0:
                raise ValueError(f"fork_seqs: source sequence {s} holds no GPU blocks")
            if not 1 <= p <= have * bs:
                raise ValueError(f"fork_seqs: length {p} outside [1, {have * bs}] for source sequence {s} ({have} blocks)")
            if on_gpu[B + i] > 0 or on_cpu[B + i] > 0:
                raise ValueError(f"fork_seqs: destination sequence {d} already holds blocks")
        if B == 0:
            return
        src_t, dst_t, lens_t = self._stage_metadata(src, dst, lens)
        gpu.fork_blocks_for_seqs(src_t, dst_t, lens_t, src_seq_ids_list=src, dst_seq_ids_list=dst, lens_list=lens)
        if any(p % bs for p in lens):
            self._wait_for_swaps()      # pending swap copies may still read or write these pages
            copy_block_tails(self.k_cache, self.v_cache, self.token_cache, gpu.block_table, src_t, dst_t, lens_t, bs)

    # ------------------------------------------------------------------ swap / free
    def _swap(self, seq_ids_list: list, is_swap_in: bool):
        """model.py:361-379, without the two `.tolist()` syncs on the allocation side: the host mirror knows the
        sizes; only the gathered / new block ids themselves have to come back for the memcpy plan."""
        src = self.cpu_block_manager if is_swap_in else self.gpu_block_manager
        dst = self.gpu_block_manager if is_swap_in else self.cpu_block_manager
        seq_ids = torch.tensor(seq_ids_list, dtype=torch.int32, device=self.device)
        nblocks = src.get_num_allocated_blocks_host(seq_ids_list)
        seq_lengths_list = [n * self.engine_config.block_size for n in nblocks]
        seq_lengths = torch.tensor(seq_lengths_list, dtype=torch.int32, device=self.device)
        src_block_ids = src.gather_allocated_blocks_and_free(seq_ids, seq_ids_list=seq_ids_list)
        dst_block_ids = dst.allocate_blocks_for_seqs(seq_ids, seq_lengths, seq_ids_list=seq_ids_list,
                                                     target_lens_list=seq_lengths_list)
        device_ids = bool(getattr(self.engine_config, "device_swap", False))
        if device_ids:
            src_ids, dst_ids = src_block_ids.to(torch.int64), dst_block_ids
        else:
            src_ids, dst_ids = src_block_ids.tolist(), dst_block_ids.tolist()
        copy = swiftllm_c.swap_blocks_device if device_ids else swiftllm_c.swap_blocks
        if not getattr(self.engine_config, "swap_on_copy_stream", False):
            # ids stay on the device (device_swap): one gather/scatter kernel over the mapped swap space, sync-free
            copy(src_ids, dst_ids, is_swap_in, self.k_cache, self.v_cache, self.k_swap, self.v_swap)
            self._swap_token_pages(copy, src_ids, dst_ids, is_swap_in)
            return
        # copy stream: the copy starts once everything enqueued so far on this stream (the block-table kernels above, the KV
        # stores of earlier steps) has finished; the next forward waits for `_swap_done` before it touches the cache
        if self._swap_stream is None:
            self._swap_stream = torch.cuda.Stream(device=self.device)
        ready = torch.cuda.Event()
        ready.record()
        with torch.cuda.stream(self._swap_stream):
            self._swap_stream.wait_event(ready)
            copy(src_ids, dst_ids, is_swap_in, self.k_cache, self.v_cache, self.k_swap, self.v_swap)
            self._swap_token_pages(copy, src_ids, dst_ids, is_swap_in)
            if device_ids and src_ids.is_cuda:       # the id tensors were allocated on the main stream
                src_ids.record_stream(self._swap_stream); dst_ids.record_stream(self._swap_stream)
            self._swap_done = torch.cuda.Event()
            self._swap_done.record()

    def _swap_token_pages(self, copy, src_ids, dst_ids, is_swap_in: bool):
        """The token pages follow their KV blocks through the same id lists, once a penalised step has run (a run without
        penalties swaps exactly what it did before).  The swap entry points move a (k, v) pair: the one table goes in as both,
        so its 4 B per token are copied twice."""
        if self._penalties_used:
            copy(src_ids, dst_ids, is_swap_in, self.token_cache, self.token_cache, self.token_swap, self.token_swap)

    @torch.inference_mode()
    def swap_in_seqs(self, seq_ids_list: list):
        """Move the blocks of the given sequences from the CPU swap space to the GPU cache."""
        self._swap(seq_ids_list, True)

    @torch.inference_mode()
    def swap_out_seqs(self, seq_ids_list: list):
        """Move the blocks of the given sequences from the GPU cache to the CPU swap space."""
        self._swap(seq_ids_list, False)

    @torch.inference_mode()
    def free_seqs_resources(self, seq_ids_list: list):
        """model.py:401-408."""
        seq_ids = torch.tensor(seq_ids_list, dtype=torch.int32, device=self.device)
        self.gpu_block_manager.free_blocks_for_seqs(seq_ids, seq_ids_list=seq_ids_list)
        self.cpu_block_manager.free_blocks_for_seqs(seq_ids, seq_ids_list=seq_ids_list)
