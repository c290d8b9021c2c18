"""Reference: swiftllm/worker/layers/post_layer.py:9-40 (last-token gather, final RMSNorm, lm_head, greedy argmax).

Addition (tensor parallelism, SURVEY.md §8 f-3): with a vocabulary-sharded lm_head every rank computes the logits of its
V / tp_size rows only and the greedy token is found with ONE all-gather of per-rank (max logit, global index) pairs
(8 bytes per sequence and rank) instead of every rank streaming the whole lm_head.

Addition (sampling, csrc/sampling.cu): when the step carries sampling parameters (infer_state.sampling) the token comes from the
sampling kernel instead of argmax.  With a sharded lm_head, batches without top-k / top-p sample each shard and exchange
(best score, global index) pairs through the same all-gather - the noise is keyed by the global index, so the merged token is
the unsharded one; otherwise the logits are all-gathered and every rank samples the full rows.

Addition (log-probabilities, csrc/logprobs.cu): when the step asks for them (infer_state.logprobs = N), the log-probability of
the chosen token and the top-N entries are computed from the same logits the token was chosen from, and the layer returns
(tokens, token logprobs, top ids, top logprobs).  With a sharded lm_head the full rows are gathered first, so every rank
chooses the token and computes identical log-probabilities from whole rows.

Addition (penalties, csrc/penalties.cu): when some row carries repetition / frequency / presence penalties (sampling.penalized),
the logits the token is chosen from are penalised first (a copy when log-probabilities are asked for: they stay those of the raw
logits) and the step's tokens are recorded in the token pages.  With a sharded lm_head the pair-merge path penalises each rank's
shard (vocab_offset) before its local choice; the gather path penalises the gathered full rows on every rank.  Every rank records
the same tokens in its own pages.  Rows with the no-repeat n-gram ban or DRY (sampling.ngram) go through the same launch, which
then also applies those (the kernel's n-gram instantiation); their result does not depend on the shard, so both paths agree.

Addition (prompt log-probabilities, csrc/prompt_logprobs.cu): when the step scores prompt rows (infer_state.prompt_logprobs),
the last-row path above runs first, unchanged; then the prompt rows go through the final RMSNorm, lm_head (gathered when
sharded, as above) and the prompt kernel in blocks of `block_rows` rows, written into slices of preallocated outputs, and the
layer returns (what the last-row path returned, (logprobs, ranks, top ids, top logprobs) of the rows).

Addition (constrained decoding, csrc/constraints.cu): when some row carries an allowed-token mask or a logit bias
(infer_state.constraints), the logits the token is chosen from are masked and biased first, ahead of the penalties (a copy when
log-probabilities are asked for: they stay those of the raw logits).  With a sharded lm_head the pair-merge path constrains each
rank's shard (vocab_offset) before its local choice - a shard with no allowed id yields a -inf pair, which the merge never picks
because the host checked that every mask allows some id; the gather path constrains the gathered full rows on every rank.

Addition (min-p, typical-p and XTC, csrc/sampling.cu): rows with these filters (sampling.truncated) are sampled by the truncated
entry with their filter views.  The filters need whole rows, so such rows count as filtered and a sharded lm_head gathers them."""
import torch
import torch.distributed as dist

from swiftllm_b200.worker.infer_state import LlamaInferState
from swiftllm_b200.worker.kernels.constraints import constrain_logits
from swiftllm_b200.worker.kernels.linear import linear
from swiftllm_b200.worker.kernels.logprobs import prompt_logprobs, token_logprobs
from swiftllm_b200.worker.kernels.penalties import apply_penalties
from swiftllm_b200.worker.kernels.rmsnorm import rmsnorm_inplace
from swiftllm_b200.worker.kernels.sampling import sample_tokens


def merge_sharded_argmax(pairs: torch.Tensor) -> torch.Tensor:
    """pairs fp32 [ranks, batch, 2] = (max logit of the rank's vocabulary shard, its GLOBAL token index) -> int64 [batch]:
    the index of the largest logit; among equal maxima the smallest index (first occurrence, the convention of
    torch.argmax over the unsharded logits, post_layer.py:39).  Indices < 2^24 are exact in fp32."""
    vals, idx = pairs[..., 0], pairs[..., 1]
    best = vals.max(dim=0).values
    cand = torch.where(vals == best, idx, torch.full_like(idx, float("inf")))
    return cand.min(dim=0).values.to(torch.int64)


class LlamaPostLayer:
    def __init__(self, model_config, weights, tp_group=None, tp_rank: int = 0, tp_size: int = 1):
        self.model_config = model_config
        self.weights = weights
        self.tp_group, self.tp_rank, self.tp_size = tp_group, tp_rank, tp_size
        self.sharded = bool(getattr(weights, "lm_head_sharded", False))
        assert model_config.vocab_size < (1 << 24) or not self.sharded
        self.last_logits = None     # kept for parity tests (the reference discards them)
        self.last_prompt_logits = None      # the scored prompt rows' logits, likewise
        self.keep_logits = False

    def forward(self, input_embds: torch.Tensor, infer_state: LlamaInferState, already_normed: bool = False):
        """`already_normed`: input_embds rows are rmsnorm(final residual) already (TP fused-exchange path; RMSNorm is
        row-wise, so normalising before or after the last-token gather is the same computation)."""
        out = self._last_rows(input_embds, infer_state, already_normed)
        if infer_state.prompt_logprobs is None:
            return out
        return out, self._prompt_rows(input_embds, infer_state.prompt_logprobs, already_normed)

    def _prompt_rows(self, input_embds: torch.Tensor, st, already_normed: bool):
        """(logprob fp32 [K], rank int32 [K], top ids int32 [K, N], top logprobs fp32 [K, N]) of the rows of st.pieces, computed
        st.block_rows rows at a time so the logits block stays within the step's memory bound.  The row and target tensors are
        built here, after the layers (device-side fills and slices of the staged ids: no host-to-device copy, no sync)."""
        K, n, dev = st.num_rows, st.top_n, input_embds.device
        ids = st.input_ids
        rows = torch.cat([torch.arange(s, s + c - 1 + (nx is not None), dtype=torch.int32, device=dev) for s, c, nx in st.pieces])
        targets = torch.cat([t for s, c, nx in st.pieces
                             for t in (ids[s + 1:s + c],) + (() if nx is None else (ids.new_full((1,), nx),))])
        assert rows.shape[0] == K and targets.shape[0] == K
        res = (torch.empty((K,), dtype=torch.float32, device=dev), torch.empty((K,), dtype=torch.int32, device=dev),
               torch.empty((K, n), dtype=torch.int32, device=dev), torch.empty((K, n), dtype=torch.float32, device=dev))
        kept = []
        for b0 in range(0, K, st.block_rows):
            b1 = min(K, b0 + st.block_rows)
            x = input_embds.index_select(0, rows[b0:b1])
            if not already_normed:
                rmsnorm_inplace(x, self.weights.final_norm, self.model_config.rms_norm_eps)
            logits = linear(x, self.weights.lm_head)
            del x
            if self.sharded:
                logits = self._gather_logits(logits)
            prompt_logprobs(logits, targets[b0:b1], n, out=tuple(t[b0:b1] for t in res))
            if self.keep_logits:
                kept.append(logits.clone())
            del logits
        if self.keep_logits:                                   # parity tests only
            self.last_prompt_logits = torch.cat(kept)
        return res

    def _last_rows(self, input_embds: torch.Tensor, infer_state: LlamaInferState, already_normed: bool):
        idx = infer_state.last_token_indices
        if idx is None:
            idx = torch.cat((
                infer_state.prefill_seq_start_locs + infer_state.prefill_seq_lens - 1,
                torch.arange(infer_state.num_prefill_tokens, infer_state.num_tokens, device=input_embds.device, dtype=torch.int32)
            ), dim=0)
        last_input = input_embds.index_select(0, idx)          # [batch_size, hidden_size], fresh contiguous buffer
        if not already_normed:
            rmsnorm_inplace(last_input, self.weights.final_norm, self.model_config.rms_norm_eps)
        logits = linear(last_input, self.weights.lm_head)      # [batch_size, vocab_size] (or this rank's V / tp_size columns)
        sp, n, con = infer_state.sampling, infer_state.logprobs, infer_state.constraints
        pen = sp is not None and sp.penalized
        sampled = sp is not None and sp.sampled
        B, Vs = logits.shape
        if not self.sharded or (sp is not None and sp.filtered) or n is not None:
            # choose the token from whole rows: top-k / top-p and log-probabilities need them, so a sharded lm_head gathers
            # them and every rank chooses the token
            full = self._gather_logits(logits) if self.sharded else logits
            if self.keep_logits:
                self.last_logits = full.clone() if pen or con is not None else full
            chosen = full if con is None else self._constrained(full, con, copy=n is not None)
            if pen:
                chosen = self._penalised(chosen, infer_state, idx, copy=n is not None and con is None)
            if sampled:
                tokens = sample_tokens(chosen, sp.temperature, sp.top_k, sp.top_p, sp.seed, sp.pos, **sp.truncation_kwargs())
            else:
                tokens = torch.argmax(chosen, dim=1)
            return tokens if n is None else (tokens,) + token_logprobs(full, tokens, n)
        raw_full = self._gather_logits(logits) if self.keep_logits and (pen or con is not None) else None
        if con is not None:
            self._constrained(logits, con, copy=False, vocab_offset=self.tp_rank * Vs)
        if pen:
            self._penalised(logits, infer_state, idx, copy=False, vocab_offset=self.tp_rank * Vs)
        if sampled:
            mine = torch.empty((B, 2), dtype=torch.float32, device=logits.device)
            sample_tokens(logits, sp.temperature, sp.top_k, sp.top_p, sp.seed, sp.pos, vocab_offset=self.tp_rank * Vs,
                          out_pairs=mine, **sp.truncation_kwargs())
        else:
            local = torch.argmax(logits, dim=1)
            mine = torch.stack((logits.gather(1, local[:, None]).squeeze(1).float(),
                                (local + self.tp_rank * Vs).float()), dim=1)             # [B, 2]
        # outputs in the concatenated form ([ranks * B, ...]): accepted by both NCCL and gloo
        pairs = torch.empty((self.tp_size * B, 2), dtype=torch.float32, device=logits.device)
        dist.all_gather_into_tensor(pairs, mine.contiguous(), group=self.tp_group)
        if self.keep_logits:                                   # parity tests only: reassemble the full logits
            self.last_logits = raw_full if raw_full is not None else self._gather_logits(logits)
        return merge_sharded_argmax(pairs.view(self.tp_size, B, 2))

    @staticmethod
    def _constrained(logits: torch.Tensor, con, copy: bool, vocab_offset: int = 0) -> torch.Tensor:
        """The masked and biased logits (in place, or a copy)."""
        out = logits.clone() if copy else logits
        constrain_logits(out, con.mask_index, con.masks, con.bias_index, con.bias_starts, con.bias_ids, con.bias_values,
                         vocab_offset=vocab_offset)
        return out

    @staticmethod
    def _penalised(logits: torch.Tensor, infer_state: LlamaInferState, last_idx: torch.Tensor, copy: bool,
                   vocab_offset: int = 0) -> torch.Tensor:
        """The penalised logits (in place, or a copy), the step's tokens recorded in the token pages."""
        sp = infer_state.sampling
        out = logits.clone() if copy else logits
        apply_penalties(out, sp.repetition_penalty, sp.frequency_penalty, sp.presence_penalty, sp.pos, infer_state.seq_ids,
                        sp.input_ids, last_idx, infer_state.prefill_seq_lens, infer_state.num_prefill_seqs, sp.block_table,
                        sp.token_cache, vocab_offset=vocab_offset, **sp.ngram_kwargs())
        return out

    def _gather_logits(self, logits: torch.Tensor) -> torch.Tensor:
        """[B, V / tp_size] shards of every rank -> [B, V] (vocabulary order)."""
        B, Vs = logits.shape
        full = torch.empty((self.tp_size * B, Vs), dtype=logits.dtype, device=logits.device)
        dist.all_gather_into_tensor(full, logits.contiguous(), group=self.tp_group)
        return full.view(self.tp_size, B, Vs).permute(1, 0, 2).reshape(B, self.tp_size * Vs)
