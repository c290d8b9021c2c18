"""Per-forward metadata handed to every kernel wrapper.

The field NAMES are the interface the reference's wrappers read (`swiftllm/worker/infer_state.py:5-29`: anything that is
called with an `infer_state` looks these attributes up), so they are kept; grouping, types and the trailing optional fields
are this implementation's.  All tensors are int32 (or the model dtype for cos/sin) on the model's device; instances are always
built with keyword arguments (worker/model.py)."""
import dataclasses
from typing import Optional

import torch


@dataclasses.dataclass
class LlamaInferState:
    # ---- the packed batch: prefill sequences first, then one row per decoding sequence
    batch_size: int                                 # sequences in the batch
    num_tokens: int                                 # rows of the activation matrix
    seq_ids: torch.Tensor                           # [batch_size] block-table row of every sequence
    num_prefill_seqs: int
    num_decoding_seqs: int
    num_prefill_tokens: int                         # rows [0, num_prefill_tokens) are prompt tokens

    # ---- prefill part
    prefill_seq_lens: torch.Tensor                  # [num_prefill_seqs] tokens of each prompt (chunk) in this batch
    prefill_seq_start_locs: torch.Tensor            # [num_prefill_seqs] first row of each prompt
    prefill_seq_start_locs_with_end: torch.Tensor   # [num_prefill_seqs + 1] the same, closed with num_prefill_tokens
    max_prefill_len: int

    # ---- decode part
    decoding_seq_lens: torch.Tensor                 # [num_decoding_seqs] sequence lengths INCLUDING the new token
    max_decoding_len: int
    seq_block_size: int                             # the reference's flash-decoding split (model.py:305-324) ...
    num_seq_blocks: int                             # ... and the number of splits of the longest sequence

    # ---- attention / rotary constants of the step
    softmax_scale: float                            # head_dim ** -0.5
    position_cos: torch.Tensor                      # [num_tokens, head_dim / 2] rows of the RoPE tables at the tokens' positions
    position_sin: torch.Tensor

    ignore_kvcache: bool                            # memory-profiling forward: no KV store, no decode attention

    # ---- additions of this implementation (defaults keep the reference's behaviour)
    # Split size the library should use for paged attention; 0 = choose v1 / v2 itself.  `seq_block_size` above can be forced
    # onto the kernel by copying it here.
    paged_attn_seq_block_size: int = 0
    last_token_indices: Optional[torch.Tensor] = None   # [batch_size] rows to sample from (post_layer.py:24-31), host-computed
    # Chunked ("prefix-aware") prefill, SURVEY.md §8 f-1: prefill entry i holds the tokens at positions
    # [prefill_prefix_lens[i], prefill_prefix_lens[i] + prefill_seq_lens[i]) of its sequence; everything before is already in
    # the KV cache.  None = whole prompts, attention over the packed k/v.
    prefill_prefix_lens: Optional[torch.Tensor] = None  # [num_prefill_seqs]
    max_prefill_kv_len: int = 0                          # max_i(prefix_i + chunk_i); 0 when not chunked
    # Speculative verification (LlamaModel.forward_speculative): the chunks are an input token plus drafts (1..8 rows), attended
    # by the multi-query verify kernel instead of the chunked-prefill kernel
    speculative: bool = False
    # Per-row sampling parameters (SamplingParams) on the device; None = greedy argmax for every row
    sampling: Optional["SamplingState"] = None
    # Top-N of the step's log-probabilities (the largest SamplingParams.logprobs of the batch); None = no log-probabilities,
    # and the post layer returns the token tensor alone
    logprobs: Optional[int] = None
    # Prompt log-probabilities (SamplingParams.prompt_logprobs): the prefill rows to score; None = none, and the post layer
    # returns what it returned before
    prompt_logprobs: Optional["PromptLogprobsState"] = None
    # Allowed-token masks and logit bias of the step's last rows (csrc/constraints.cu); None = no row is constrained.  Kept apart
    # from `sampling`: a constrained step may be greedy with no sampling parameters at all
    constraints: Optional["ConstraintState"] = None
    # Per-request LoRA adapters (worker/lora.py, csrc/lora.cu): the slot pool and the step's tile list; None = no row is adapted
    lora: Optional["LoraState"] = None


@dataclasses.dataclass
class LoraState:
    pool: object                    # worker.lora.LoraPool
    tiles: torch.Tensor             # [num_tiles, 3] int32 (first row, rows, slot); rows 0 pads a graph's fixed tile count


@dataclasses.dataclass
class PromptLogprobsState:
    # host ints, one per asking entry with rows to score, in batch order: (first row in the activation matrix, token count n,
    # id of the prompt token after the entry or None).  Its rows are [first, first + n - 1), plus the last one with a next id;
    # row r scores input_ids[r + 1], the last row the next id.  The device tensors are built by the post layer after the layers,
    # so the prompt part allocates nothing while the forward's activations are live.
    pieces: list
    num_rows: int                   # K, the rows to score
    input_ids: torch.Tensor         # [num_tokens] int32 the step's staged input ids
    top_n: int                      # the largest prompt_logprobs of the asking entries
    block_rows: int                 # rows per lm_head + log-probability block (bounds the step's extra memory)


@dataclasses.dataclass
class SamplingState:
    temperature: torch.Tensor       # [batch_size] float32, 0 = greedy row
    top_k: torch.Tensor             # [batch_size] int32
    top_p: torch.Tensor             # [batch_size] float32
    seed: torch.Tensor              # [batch_size] int64
    pos: torch.Tensor               # [batch_size] int32: sequence length after this step's input (noise counter)
    filtered: bool                  # some row uses top-k or top-p (needs the whole vocabulary row on one rank)
    # ---- penalties (csrc/penalties.cu); None when no row of the step has any
    repetition_penalty: Optional[torch.Tensor] = None   # [batch_size] float32, 1 = off
    frequency_penalty: Optional[torch.Tensor] = None    # [batch_size] float32, 0 = off
    presence_penalty: Optional[torch.Tensor] = None     # [batch_size] float32, 0 = off
    # ---- n-gram ban and DRY (csrc/penalties.cu); None when no row of the step has them (then the penalties above are staged too)
    no_repeat_ngram_size: Optional[torch.Tensor] = None     # [batch_size] int32, 0 = off
    dry_allowed_length: Optional[torch.Tensor] = None       # [batch_size] int32
    dry_multiplier: Optional[torch.Tensor] = None           # [batch_size] float32, 0 = off
    dry_base: Optional[torch.Tensor] = None                 # [batch_size] float32
    dry_breakers: Optional[torch.Tensor] = None             # [batch_size, 16] int32, -1 = unused
    # ---- min-p, typical-p and XTC (csrc/sampling.cu, the truncated entry); None when no sampled row of the step has them
    min_p: Optional[torch.Tensor] = None                    # [batch_size] float32, 0 = off
    typical_p: Optional[torch.Tensor] = None                # [batch_size] float32, 1 = off
    xtc_threshold: Optional[torch.Tensor] = None            # [batch_size] float32
    xtc_probability: Optional[torch.Tensor] = None          # [batch_size] float32, 0 = off
    sampled: bool = True            # some row has temperature > 0; False: every row takes the argmax of its penalised logits
    # the token history the penalty kernel reads and extends, set by the model: the step's input ids (int32 [num_tokens]), the
    # block table and the token pages (int32 [num_blocks, block_size])
    input_ids: Optional[torch.Tensor] = None
    block_table: Optional[torch.Tensor] = None
    token_cache: Optional[torch.Tensor] = None

    @property
    def penalized(self) -> bool:
        return self.repetition_penalty is not None

    @property
    def ngram(self) -> bool:
        return self.no_repeat_ngram_size is not None

    @property
    def truncated(self) -> bool:
        return self.min_p is not None

    def truncation_kwargs(self) -> dict:
        """The filter keyword arguments of worker.kernels.sampling.sample_tokens ({} without them)."""
        if not self.truncated:
            return {}
        return dict(min_p=self.min_p, typical_p=self.typical_p, xtc_threshold=self.xtc_threshold,
                    xtc_probability=self.xtc_probability)

    def ngram_kwargs(self) -> dict:
        """The n-gram keyword arguments of worker.kernels.penalties.apply_penalties ({} without n-gram controls)."""
        if not self.ngram:
            return {}
        return dict(no_repeat_ngram_size=self.no_repeat_ngram_size, dry_allowed_length=self.dry_allowed_length,
                    dry_multiplier=self.dry_multiplier, dry_base=self.dry_base, dry_breakers=self.dry_breakers)

    @staticmethod
    def from_staged(words: torch.Tensor, pos: torch.Tensor, filtered: bool, sampled: bool = True,
                    truncated: bool = False) -> "SamplingState":
        """`words`: the int32 device view staged from swiftllm_b200.sampling_params.sampling_words (8-byte aligned); 8 * B
        words carry the penalties after the 5 * B sampling words; 28 * B words also the n-gram controls after those.
        `truncated` (sampling_params.has_truncation): the last 4 * B words are the min-p, typical-p and XTC parameters."""
        B = pos.shape[0]
        pen = {}
        if truncated:
            t = words[words.shape[0] - 4 * B:].view(torch.float32)
            pen = dict(min_p=t[:B], typical_p=t[B:2 * B], xtc_threshold=t[2 * B:3 * B], xtc_probability=t[3 * B:])
            words = words[:words.shape[0] - 4 * B]
        if words.shape[0] in (8 * B, 28 * B):
            pen.update(repetition_penalty=words[5 * B:6 * B].view(torch.float32),
                       frequency_penalty=words[6 * B:7 * B].view(torch.float32),
                       presence_penalty=words[7 * B:8 * B].view(torch.float32))
        if words.shape[0] == 28 * B:
            pen.update(no_repeat_ngram_size=words[8 * B:9 * B], dry_allowed_length=words[9 * B:10 * B],
                       dry_multiplier=words[10 * B:11 * B].view(torch.float32), dry_base=words[11 * B:12 * B].view(torch.float32),
                       dry_breakers=words[12 * B:28 * B].view(B, 16))
        return SamplingState(temperature=words[2 * B:3 * B].view(torch.float32), top_k=words[3 * B:4 * B],
                             top_p=words[4 * B:5 * B].view(torch.float32), seed=words[:2 * B].view(torch.int64), pos=pos,
                             filtered=filtered, sampled=sampled, **pen)


@dataclasses.dataclass
class ConstraintState:
    """Device views of the staged constraint region (swiftllm_b200.sampling_params.constraint_words), one row per last row."""
    mask_index: torch.Tensor        # [rows] int32: row of `masks`, -1 = no mask
    masks: torch.Tensor             # [num_masks, W] int32 bit words of global ids
    bias_index: torch.Tensor        # [rows] int32: bias entry, -1 = no bias
    bias_starts: torch.Tensor       # [num_entries + 1] int32 CSR starts
    bias_ids: torch.Tensor          # [num_bias] int32 global ids (-1: padding, matches no id)
    bias_values: torch.Tensor       # [num_bias] float32

    @staticmethod
    def from_staged(words: torch.Tensor, num_rows: int, num_masks: int, mask_words: int, num_entries: int,
                    num_bias: int) -> "ConstraintState":
        R, E, NB = num_rows, num_entries, num_bias
        o = [0, R, 2 * R, 2 * R + E + 1, 2 * R + E + 1 + NB, 2 * R + E + 1 + 2 * NB]
        assert words.shape[0] == o[5] + num_masks * mask_words
        return ConstraintState(mask_index=words[:o[1]], bias_index=words[o[1]:o[2]], bias_starts=words[o[2]:o[3]],
                               bias_ids=words[o[3]:o[4]], bias_values=words[o[4]:o[5]].view(torch.float32),
                               masks=words[o[5]:].view(num_masks, mask_words))
