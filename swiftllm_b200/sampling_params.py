"""Per-request sampling parameters and log-probability results (new: the reference decodes greedily only)."""
import dataclasses
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

MAX_LOGPROBS = 20                   # csrc/logprobs.cu: kMaxTopN
MAX_LOGIT_BIAS = 1024               # entries of SamplingParams.logit_bias (csrc/constraints.cu reads them per row)
MAX_BIAS = 100.0                    # |logit_bias value| bound of the OpenAI API


@dataclasses.dataclass
class SamplingParams:
    """temperature 0 is greedy decoding (top_k / top_p ignored).  top_k 0 and top_p 1 switch those filters off; tokens tied
    with the last one kept by either filter are kept too.  seed None draws a fresh seed from the model's generator
    (EngineConfig.sampling_seed), so runs are reproducible while repeated prompts still vary; a fixed seed makes the token a
    function of the logits, the parameters and the sequence length only.

    logprobs (LlamaModel.forward_with_logprobs): None returns none, 0 the returned token's log-probability, 1..20 also the
    top-N alternatives.  They are log_softmax of the raw logits - the model's distribution before penalties, temperature, top-k and
    top-p; a penalised greedy token therefore need not be top[0].  forward / forward_async ignore the field.

    prompt_logprobs (LlamaModel.forward_with_logprobs, prefill entries): None returns none, 0 the log-probability and rank of
    every scored prompt token, 1..20 also its top-N alternatives (PromptLogprobs), of the same raw distribution.  It changes
    neither the staged sampling words nor the tokens; forward / forward_async / forward_speculative ignore it.

    Penalties (csrc/penalties.cu; the order and formulas of vLLM), applied to the logits before greedy argmax or sampling, in fp32:
    repetition_penalty r (1: off) divides a positive logit / multiplies a non-positive one of every token seen in the prompt or
    the output; then frequency_penalty f and presence_penalty p (0: off) subtract f * count + p from every token that occurs
    count > 0 times in the output.  The history is read from the token pages the model records in steps where a row carries
    penalties, so a request that uses them must pass the same SamplingParams from its first prefill chunk on.

    logit_bias (csrc/constraints.cu): None or {token id: bias}, at most MAX_LOGIT_BIAS entries, biases finite in [-100, 100], ids
    in [0, vocab_size) (checked by the step).  Applied after the step's allowed-token mask (token_masks_list of LlamaModel.forward)
    and before the penalties: l = round(float(l) + bias), one fp32 add and one rounding to the storage dtype; a masked id stays
    -inf.  Log-probabilities stay those of the raw logits."""
    temperature: float = 0.0
    top_k: int = 0
    top_p: float = 1.0
    seed: Optional[int] = None
    logprobs: Optional[int] = None
    prompt_logprobs: Optional[int] = None
    repetition_penalty: float = 1.0
    frequency_penalty: float = 0.0
    presence_penalty: float = 0.0
    logit_bias: Optional[dict] = None

    def validate(self):
        if not (isinstance(self.temperature, (int, float)) and math.isfinite(self.temperature) and self.temperature >= 0):
            raise ValueError(f"temperature must be a finite number >= 0, got {self.temperature!r}")
        if isinstance(self.top_k, bool) or not isinstance(self.top_k, (int, np.integer)) or not 0 <= self.top_k < 2 ** 31:
            raise ValueError(f"top_k must be an integer in [0, 2^31), got {self.top_k!r}")
        if not (isinstance(self.top_p, (int, float)) and 0 < self.top_p <= 1):
            raise ValueError(f"top_p must be in (0, 1], got {self.top_p!r}")
        if self.seed is not None and (isinstance(self.seed, bool) or not isinstance(self.seed, (int, np.integer))
                                      or not 0 <= self.seed < 2 ** 64):
            raise ValueError(f"seed must be None or an integer in [0, 2^64), got {self.seed!r}")
        for name in ("logprobs", "prompt_logprobs"):
            v = getattr(self, name)
            if v is not None and (isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= v <= MAX_LOGPROBS):
                raise ValueError(f"{name} must be None or an integer in [0, {MAX_LOGPROBS}], got {v!r}")
        if not (_is_real(self.repetition_penalty) and math.isfinite(self.repetition_penalty) and self.repetition_penalty > 0):
            raise ValueError(f"repetition_penalty must be a finite number > 0, got {self.repetition_penalty!r}")
        for name in ("frequency_penalty", "presence_penalty"):
            v = getattr(self, name)
            if not (_is_real(v) and math.isfinite(v) and -2 <= v <= 2):
                raise ValueError(f"{name} must be a finite number in [-2, 2], got {v!r}")
        lb = self.logit_bias
        if lb is not None:
            if not isinstance(lb, dict):
                raise ValueError(f"logit_bias must be None or a dict {{token id: bias}}, got {type(lb).__name__}")
            if len(lb) > MAX_LOGIT_BIAS:
                raise ValueError(f"logit_bias has {len(lb)} entries; at most {MAX_LOGIT_BIAS} are supported")
            for k, v in lb.items():
                if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= k < 2 ** 31:
                    raise ValueError(f"logit_bias keys must be token ids (integers >= 0), got {k!r}")
                if not (_is_real(v) and math.isfinite(v) and -MAX_BIAS <= v <= MAX_BIAS):
                    raise ValueError(f"logit_bias values must be finite numbers in [-100, 100], got {v!r} for id {k}")

    def has_penalties(self) -> bool:
        return self.repetition_penalty != 1.0 or self.frequency_penalty != 0.0 or self.presence_penalty != 0.0


def _is_real(v) -> bool:
    return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool)


class PromptLogprobs(NamedTuple):
    """The scored prompt tokens of one prefill entry (SamplingParams.prompt_logprobs).  An entry at prefix p holding tokens
    x_p .. x_{p+n-1} scores x_{p+1} .. x_{p+n-1}, and the next prompt token when the caller passes it: k = n - 1 (+ 1) tokens at
    positions first_position = p + 1 onwards (position 0 is never scored).  Row j: token_ids[j], its log-probability under the
    raw model distribution given the tokens before it, its rank (1 + the number of ids with a larger logit; 1 for the greedy
    token) and the N most likely ids with their log-probabilities, ordered by (logprob desc, id asc)."""
    first_position: int
    token_ids: np.ndarray           # int64 [k]
    logprobs: np.ndarray            # float32 [k]
    ranks: np.ndarray               # int32 [k]
    top_ids: np.ndarray             # int32 [k, N]
    top_logprobs: np.ndarray        # float32 [k, N]


class TokenLogprobs(NamedTuple):
    """One batch entry of LlamaModel.forward_with_logprobs.  logprob: log-probability of `token` under the raw model
    distribution (log_softmax of the logits); top: [(token id, logprob)] of the N most likely tokens, most likely first, ties
    broken by the smaller id (the empty list for logprobs=0).  Both None when the entry did not ask.  prompt: the entry's
    PromptLogprobs when it is a prefill entry with SamplingParams.prompt_logprobs set, else None."""
    token: int
    logprob: Optional[float] = None
    top: Optional[list] = None
    prompt: Optional[PromptLogprobs] = None


def logprobs_top_n(params_list: Optional[list]) -> Optional[int]:
    """The per-launch N: the largest `logprobs` of the (validated) list, None when no entry asks."""
    asked = [int(sp.logprobs) for sp in params_list or [] if sp.logprobs is not None]
    return max(asked) if asked else None


def prompt_logprobs_top_n(params_list: Optional[list]) -> Optional[int]:
    """The per-launch N of the prompt rows: the largest `prompt_logprobs` of the (validated) list, None when no entry asks."""
    asked = [int(sp.prompt_logprobs) for sp in params_list or [] if sp.prompt_logprobs is not None]
    return max(asked) if asked else None


def _i32(words: np.ndarray) -> list:
    return words.astype(np.uint32).view(np.int32).tolist()


def sampling_words(params_list: list, batch_size: int, rng: np.random.Generator):
    """Validates the list and returns the staged int32 words (seed lo/hi interleaved [2B], temperature bits [B], top_k [B],
    top_p bits [B], and when some row has penalties the fp32 bits of repetition, frequency and presence penalty [3B]) and whether
    any row filters (top-k / top-p); None when every row is greedy and none has penalties.  Raises ValueError."""
    if len(params_list) != batch_size:
        raise ValueError(f"sampling_params_list has {len(params_list)} entries for a batch of {batch_size}")
    for sp in params_list:
        if not isinstance(sp, SamplingParams):
            raise ValueError(f"sampling_params_list entries must be SamplingParams, got {type(sp).__name__}")
        sp.validate()
    # a fresh seed for every unseeded row, drawn even for greedy rows so the stream does not depend on the batch's mix
    seeds = np.array([int(rng.integers(0, 2 ** 63)) if sp.seed is None else int(sp.seed) for sp in params_list], dtype=np.uint64)
    penalized = any(sp.has_penalties() for sp in params_list)
    if not penalized and all(sp.temperature == 0 for sp in params_list):
        return None
    temp = np.array([sp.temperature for sp in params_list], dtype=np.float32)
    top_p = np.array([sp.top_p for sp in params_list], dtype=np.float32)
    top_k = [int(sp.top_k) for sp in params_list]
    filtered = any(sp.temperature > 0 and (sp.top_k > 0 or sp.top_p < 1) for sp in params_list)
    words = _i32(seeds.view(np.uint32)) + _i32(temp.view(np.uint32)) + top_k + _i32(top_p.view(np.uint32))
    if penalized:
        for name in ("repetition_penalty", "frequency_penalty", "presence_penalty"):
            words += _i32(np.array([getattr(sp, name) for sp in params_list], dtype=np.float32).view(np.uint32))
    return words, filtered


def has_penalties(params_list: Optional[list]) -> bool:
    """Some entry of the (validated) list has a penalty: the step applies them and records its tokens in the token pages."""
    return any(sp.has_penalties() for sp in params_list or [])


def token_mask(vocab_size: int, allowed_ids) -> np.ndarray:
    """The packed mask (int32 [ceil(vocab_size / 32)], the layout of xgrammar and vLLM) that allows exactly `allowed_ids`: bit
    v % 32 of word v // 32 set.  Bits past vocab_size stay 0; they are ignored, so ~token_mask(V, ids) bans `ids`."""
    if isinstance(vocab_size, bool) or not isinstance(vocab_size, (int, np.integer)) or vocab_size <= 0:
        raise ValueError(f"vocab_size must be a positive integer, got {vocab_size!r}")
    ids = np.asarray(list(allowed_ids) if not isinstance(allowed_ids, np.ndarray) else allowed_ids).reshape(-1)
    if ids.size and (ids.dtype.kind not in "iu" or ids.min() < 0 or ids.max() >= vocab_size):
        raise ValueError(f"allowed_ids must be integer token ids in [0, {vocab_size})")
    words = np.zeros(((vocab_size + 31) // 32,), dtype=np.uint32)
    ids = ids.astype(np.int64)
    np.bitwise_or.at(words, ids >> 5, (np.uint32(1) << (ids & 31).astype(np.uint32)))
    return words.view(np.int32)


class ConstraintWords(NamedTuple):
    """The staged constraint region of a step (constraint_words) and the sizes that slice it: int32 words mask_index [num_rows],
    bias_index [num_rows], bias_starts [num_entries + 1], bias_ids [num_bias], bias_values fp32 bits [num_bias], masks
    [num_masks * mask_words]."""
    words: np.ndarray
    num_rows: int
    num_masks: int
    mask_words: int
    num_entries: int
    num_bias: int

    @staticmethod
    def size(num_rows: int, num_masks: int, mask_words: int, num_entries: int, num_bias: int) -> int:
        return 2 * num_rows + num_entries + 1 + 2 * num_bias + num_masks * mask_words


def _mask_rows(mask, n_rows: int, W: int, where: str, speculative: bool) -> np.ndarray:
    """A caller mask of the right type and shape as uint32 [n_rows, W] (a view where possible)."""
    if isinstance(mask, torch.Tensor):
        if mask.device.type != "cpu":
            raise ValueError(f"{where} must be a numpy array or a CPU tensor, got a tensor on {mask.device}")
        if mask.dtype not in (torch.int32, torch.uint32):
            raise ValueError(f"{where} must be int32 or uint32, got {mask.dtype}")
        mask = mask.contiguous().view(torch.int32).numpy()
    if not isinstance(mask, np.ndarray):
        raise ValueError(f"{where} must be None, a numpy array or a CPU tensor, got {type(mask).__name__}")
    if mask.dtype not in (np.int32, np.uint32):
        raise ValueError(f"{where} must be int32 or uint32, got {mask.dtype}")
    want = (n_rows, W) if speculative else (W,)
    if mask.shape != want:
        raise ValueError(f"{where} has shape {mask.shape}; expected {want} (ceil(vocab_size / 32) = {W} words per row)")
    return mask.view(np.uint32).reshape(n_rows, W)


def constraint_words(token_masks_list: Optional[list], params_list: Optional[list], batch_size: int, vocab_size: int,
                     rows: Optional[list] = None, graph: bool = False) -> Optional[ConstraintWords]:
    """The staged constraint region of a step from the caller's masks (one entry per batch entry: None or a packed int32 / uint32
    mask of W = ceil(vocab_size / 32) words; with `rows`, the per-entry row counts of a speculative step, None or [rows_i, W]) and
    the (validated) parameters' logit_bias; None when nothing is constrained.  Row r of entry i gets the entry's bias (index i).
    graph: the sizes of a captured graph - one mask slot per row (mask index = row) and the bias arrays padded to a power of two
    with ids -1, which match no token.  Raises ValueError."""
    speculative = rows is not None
    rows = [1] * batch_size if rows is None else list(rows)
    if token_masks_list is not None and len(token_masks_list) != batch_size:
        raise ValueError(f"token_masks_list has {len(token_masks_list)} entries for a batch of {batch_size}")
    W = (vocab_size + 31) // 32
    masks = [None] * batch_size if token_masks_list is None else [
        None if m is None else _mask_rows(m, n, W, f"token_masks_list[{i}]", speculative)
        for i, (m, n) in enumerate(zip(token_masks_list, rows))]
    biases = [None] * batch_size
    for i, sp in enumerate(params_list or []):
        if sp.logit_bias:
            ids = np.array(sorted(int(k) for k in sp.logit_bias), dtype=np.int64)
            if ids[-1] >= vocab_size:
                raise ValueError(f"sampling_params_list[{i}].logit_bias has token id {int(ids[-1])} outside [0, {vocab_size})")
            biases[i] = (ids.astype(np.int32), np.array([sp.logit_bias[k] for k in sorted(sp.logit_bias, key=int)], np.float32))
    if all(m is None for m in masks) and all(b is None for b in biases):
        return None
    R, E = sum(rows), batch_size
    row_entry = np.repeat(np.arange(E), rows)
    first_row = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64)
    counts = [0 if b is None else b[0].shape[0] for b in biases]
    total = sum(counts)
    NB = (0 if total == 0 else 1 << (total - 1).bit_length()) if graph else total
    M = R if graph else sum(m.shape[0] for m in masks if m is not None)
    # one buffer, written in place: mask_index, bias_index, bias_starts, bias_ids, bias_values, masks
    words = np.empty((ConstraintWords.size(R, M, W, E, NB),), dtype=np.int32)
    mask_index, bias_index = words[:R], words[R:2 * R]
    starts = words[2 * R:2 * R + E + 1]
    bias_ids = words[2 * R + E + 1:2 * R + E + 1 + NB]
    bias_vals = words[2 * R + E + 1 + NB:2 * R + E + 1 + 2 * NB].view(np.float32)
    mask_words = words[2 * R + E + 1 + 2 * NB:].view(np.uint32).reshape(M, W)
    mask_index[:] = -1
    if graph:
        mask_words[:] = 0
    k = 0
    for i, m in enumerate(masks):
        if m is not None:
            r = first_row[i] + np.arange(rows[i])
            mask_index[r] = r if graph else k + np.arange(rows[i])
            mask_words[mask_index[r]] = m
            k += rows[i]
    tail = np.uint32(0xffffffff) if vocab_size % 32 == 0 else np.uint32((1 << (vocab_size % 32)) - 1)
    live = (np.bitwise_or.reduce(mask_words[:, :-1], axis=1) != 0) | ((mask_words[:, -1] & tail) != 0)
    dead = ~live[mask_index[mask_index >= 0]]
    if dead.any():
        r = int(np.flatnonzero(mask_index >= 0)[int(np.argmax(dead))])
        i = int(row_entry[r])
        raise ValueError(f"token_masks_list[{i}] allows no token id in [0, {vocab_size})" +
                         (f" (row {r - int(first_row[i])})" if speculative else ""))
    bias_index[:] = np.where([biases[e] is not None for e in row_entry], row_entry, -1)
    starts[:] = np.concatenate([[0], np.cumsum(counts)])
    bias_ids[:] = -1
    bias_vals[:] = 0
    for i, b in enumerate(biases):
        if b is not None:
            bias_ids[starts[i]:starts[i + 1]], bias_vals[starts[i]:starts[i + 1]] = b
    return ConstraintWords(words, R, M, W, batch_size, NB)
