"""Per-request sampling parameters and log-probability results (new: the reference decodes greedily only)."""
import dataclasses
import math
from typing import NamedTuple, Optional

import numpy as np

MAX_LOGPROBS = 20                   # csrc/logprobs.cu: kMaxTopN


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
    penalties, so a request that uses them must pass the same SamplingParams from its first prefill chunk on."""
    temperature: float = 0.0
    top_k: int = 0
    top_p: float = 1.0
    seed: Optional[int] = None
    logprobs: Optional[int] = None
    prompt_logprobs: Optional[int] = None
    repetition_penalty: float = 1.0
    frequency_penalty: float = 0.0
    presence_penalty: float = 0.0

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
