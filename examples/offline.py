#!/usr/bin/env python
"""Data-plane-only generation with swiftllm_b200.LlamaModel - the counterpart of the reference's examples/offline.py (same
worker API and call order: load_weights -> profile_num_blocks -> init_kvcache_and_swap -> forward for the prompts -> forward
per generated token).  Needs an H100 (there is no CPU path).

    python examples/offline.py --model-path /data/Llama-3-8B            # real checkpoint + its HF tokenizer
    python examples/offline.py --synthetic llama3-8b                     # seeded random weights, random token ids
    ... --chunk 512        prefill the prompts in 512-token chunks through the paged cache (prefill_prefix_lens_list)
    ... --cuda-graph       replay decode steps from CUDA graphs
    ... --temperature 0.8 --top-p 0.95 [--top-k 50] [--seed 1]    sample instead of greedy decoding
    ... --logprobs 5       print each generated token's log-probability and the 5 most likely tokens (forward_with_logprobs)
    ... --prompt-logprobs 3    print each prompt's perplexity and the 3 most likely tokens at its first positions
    ... --repetition-penalty 1.1 --frequency-penalty 0.5 --presence-penalty 0.3    discourage repeats (vLLM's definitions)
    ... --speculate 4      speculative decoding: verify up to 4 prompt-lookup drafts per step (forward_speculative)
    ... --n 4 --temperature 0.8    4 samples per prompt: each prompt is prefilled once and forked 3 times (fork_seqs)
    ... --lora /data/my-adapter    run every prompt under a PEFT LoRA adapter (load_lora, lora_ids_list)
    ... --quantization fp8 e4m3 projection weights (16-bit checkpoints are quantized at load; FP8 checkpoints load as they are)
"""
import argparse
import dataclasses
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import swiftllm_b200  # noqa: E402


def prompt_lookup(tokens: list, k: int, max_ngram: int = 3) -> list:
    """Up to k draft tokens: what followed the most recent earlier occurrence of the longest suffix n-gram (n <= max_ngram) of
    `tokens`; none when no suffix recurs."""
    for n in range(min(max_ngram, len(tokens) - 1), 0, -1):
        tail = tokens[-n:]
        for s in range(len(tokens) - n - 1, -1, -1):
            if tokens[s:s + n] == tail:
                return tokens[s + n:s + n + k]
    return []


def with_adapter(model, slot: int):
    """Every forward call of `model` runs its whole batch under LoRA adapter `slot`, except the memory-profiling forward
    (ignore_kvcache=True, which takes no adapter): it runs the base model, whose activations are the same size."""
    for name in ("forward", "forward_with_logprobs", "forward_speculative"):
        def call(ids, *a, _f=getattr(model, name), **kw):
            if kw.get("ignore_kvcache"):
                return _f(ids, *a, **kw)
            return _f(ids, *a, lora_ids_list=[slot] * len(ids), **kw)
        setattr(model, name, call)


def generate(model, input_ids, new_tokens: int, chunk: int = 0, params=None, logs=None, speculate: int = 0, n: int = 1,
             prompt_logs=None):
    """Generation for a batch of prompts (sequence i uses block-table row i), greedy unless `params` (one
    swiftllm_b200.SamplingParams for every sequence) is given.  chunk > 0: the prompts are prefilled `chunk` tokens at a time
    through the paged cache.  speculate > 0: decoding verifies up to that many prompt-lookup drafts per step
    (forward_speculative); the tokens are the ones plain decoding returns.  Returns (token lists, prefill seconds, decode seconds).
    With params.logprobs set, logs[i] (a list per sequence) receives the TokenLogprobs of every generated token.  With
    params.prompt_logprobs set, prompt_logs[i] (a list per prompt) receives the PromptLogprobs of each of its prefill calls: with
    chunks, each call passes the next chunk's first token, so together they score positions 1 .. len - 1.

    n > 1: n samples per prompt.  Each prompt is prefilled once into row i; rows len(input_ids) + i * (n - 1) + j (j < n - 1)
    fork its first len - 1 tokens (fork_seqs: the full blocks are shared) and draw their own first token from the last prompt
    token, fed as a one-token prefill chunk so that penalties count it as a prompt token, as in row i.  Sample k of a prompt uses seed params.seed + k (seed None: a fresh seed per row and step), so the samples differ; the
    n * len(input_ids) sequences then decode in one batch.  Outputs and logs follow the rows: prompts first, then the forks."""
    P = len(input_ids)
    seq_ids = list(range(P))
    kids = [(i, P + i * (n - 1) + j, j + 1) for i in range(P) for j in range(n - 1)]     # (prompt, row, sample index)
    if kids and min(len(p) for p in input_ids) < 2:
        raise ValueError("n > 1 forks len - 1 prompt tokens: every prompt needs at least 2 tokens")
    row_params = [params] * P + [params if params is None or params.seed is None else
                                 dataclasses.replace(params, seed=(params.seed + k) % 2 ** 64) for _, _, k in kids]
    sp = (lambda rows: None) if params is None else (lambda rows: [row_params[i] for i in rows])
    want_lp = params is not None and (params.logprobs is not None or params.prompt_logprobs is not None)
    logs = logs if logs is not None else [[] for _ in range(P * n)]
    prompt_logs = prompt_logs if prompt_logs is not None else [[] for _ in range(P)]

    def step(*args, prompt_next_ids_list=None, **kw):
        if not want_lp:
            return model.forward(*args, **kw)
        return model.forward_with_logprobs(*args, prompt_next_ids_list=prompt_next_ids_list, **kw)
    t0 = time.perf_counter()
    if chunk > 0:                      # every call carries the next chunk of each unfinished prompt
        done = [0] * len(input_ids)
        last = [None] * len(input_ids)
        while any(d < len(p) for d, p in zip(done, input_ids)):
            live = [i for i in seq_ids if done[i] < len(input_ids[i])]
            nxt = [input_ids[i][done[i] + chunk] if done[i] + chunk < len(input_ids[i]) else None for i in live]
            toks = step([input_ids[i][done[i]:done[i] + chunk] for i in live], live, [],
                        prefill_prefix_lens_list=[done[i] for i in live], sampling_params_list=sp(live), prompt_next_ids_list=nxt)
            for i, t in zip(live, toks):
                if want_lp and t.prompt is not None:
                    prompt_logs[i].append(t.prompt)
                done[i] = min(len(input_ids[i]), done[i] + chunk)
                if done[i] == len(input_ids[i]):
                    last[i] = t             # the token sampled after the LAST chunk is the first generated token
    else:
        last = step(input_ids, seq_ids, [], sampling_params_list=sp(seq_ids))
        for i, t in enumerate(last if want_lp else []):
            if t.prompt is not None:
                prompt_logs[i].append(t.prompt)
    if kids:
        rows = [r for _, r, _ in kids]
        model.fork_seqs([i for i, _, _ in kids], rows, [len(input_ids[i]) - 1 for i, _, _ in kids])
        last = list(last) + list(step([[input_ids[i][-1]] for i, _, _ in kids], rows, [],
                                      prefill_prefix_lens_list=[len(input_ids[i]) - 1 for i, _, _ in kids],
                                      sampling_params_list=sp(rows)))
        input_ids = list(input_ids) + [input_ids[i] for i, _, _ in kids]
        seq_ids = seq_ids + rows
    if want_lp:
        for lg, r in zip(logs, last):
            lg.append(r)
        last = [r.token for r in last]
    t_prefill = time.perf_counter() - t0
    outputs = [[t] for t in last]
    seq_lens = [len(p) for p in input_ids]
    t0 = time.perf_counter()
    if speculate > 0:                  # every call verifies up to `speculate` prompt-lookup drafts per unfinished sequence
        while any(len(o) < new_tokens for o in outputs):
            live = [i for i in seq_ids if len(outputs[i]) < new_tokens]
            entries = [[outputs[i][-1]] + prompt_lookup(input_ids[i] + outputs[i], min(speculate, new_tokens - len(outputs[i]) - 1))
                       for i in live]
            res = model.forward_speculative(entries, live, [seq_lens[i] for i in live], sampling_params_list=sp(live))
            for i, r in zip(live, res):
                outputs[i] += r
                seq_lens[i] += len(r)
        return outputs, t_prefill, time.perf_counter() - t0
    for _ in range(new_tokens - 1):
        seq_lens = [n + 1 for n in seq_lens]
        last = step([[t] for t in last], seq_ids, seq_lens, sampling_params_list=sp(seq_ids))
        if want_lp:
            for lg, r in zip(logs, last):
                lg.append(r)
            last = [r.token for r in last]
        for o, t in zip(outputs, last):
            o.append(t)
    return outputs, t_prefill, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--model-path", type=str, help="directory with config.json + safetensors / pytorch_model.bin + tokenizer")
    src.add_argument("--synthetic", type=str, choices=["llama3-8b", "llama3-70b"], help="architecture to fill with seeded random weights")
    ap.add_argument("--dtype", type=str, default="bfloat16", choices=["float16", "bfloat16"])
    ap.add_argument("--new-tokens", type=int, default=20)
    ap.add_argument("--chunk", type=int, default=0, help="chunked prefill: tokens of each prompt per forward call (0 = whole prompts)")
    ap.add_argument("--cuda-graph", action="store_true")
    ap.add_argument("--temperature", type=float, default=0.0, help="0 = greedy decoding")
    ap.add_argument("--top-k", type=int, default=0, help="keep the k most likely tokens (0 = off)")
    ap.add_argument("--top-p", type=float, default=1.0, help="keep the smallest set of tokens with this much mass (1 = off)")
    ap.add_argument("--seed", type=int, default=None, help="sampling seed (default: a fresh one per step from the engine's generator)")
    ap.add_argument("--logprobs", type=int, default=None, help="print each token's log-probability and the N most likely tokens (0..20)")
    ap.add_argument("--prompt-logprobs", type=int, default=None,
                    help="print each prompt's perplexity and the N most likely tokens at its first positions (0..20)")
    ap.add_argument("--repetition-penalty", type=float, default=1.0, help="divide / multiply the logits of seen tokens (1 = off)")
    ap.add_argument("--frequency-penalty", type=float, default=0.0, help="subtract this times each token's output count (0 = off)")
    ap.add_argument("--presence-penalty", type=float, default=0.0, help="subtract this from every token already output (0 = off)")
    ap.add_argument("--speculate", type=int, default=0, help="verify up to K (<= 7) prompt-lookup drafts per decode step (0 = off)")
    ap.add_argument("--n", type=int, default=1, help="samples per prompt: prefill once, fork n - 1 times, distinct seeds (1 = off)")
    ap.add_argument("--lora", type=str, default=None, help="PEFT LoRA adapter directory: every prompt runs under this adapter")
    ap.add_argument("--quantization", type=str, default=None, choices=["fp8"],
                    help="fp8: e4m3 projection weights, 16-bit checkpoints quantized at load (default: follow the checkpoint)")
    args = ap.parse_args()
    if args.n < 1:
        ap.error("--n takes a positive number of samples")
    if not 0 <= args.speculate <= 7:
        ap.error("--speculate takes 0..7 drafts")
    if args.speculate and (args.logprobs is not None or args.prompt_logprobs is not None or args.repetition_penalty != 1.0 or args.frequency_penalty != 0.0
                           or args.presence_penalty != 0.0):
        ap.error("--speculate does not combine with --logprobs, --prompt-logprobs or penalties")

    ec = swiftllm_b200.EngineConfig(model_path=args.model_path or "", use_dummy=False, block_size=16, gpu_mem_utilization=0.9,
                                    num_cpu_blocks=0, max_seqs_in_block_table=128, max_blocks_per_seq=2048, max_batch_size=16,
                                    max_tokens_in_batch=2048 * 16, dtype=args.dtype, use_cuda_graph=args.cuda_graph,
                                    quantization=args.quantization)
    if args.lora:
        with open(os.path.join(args.lora, "adapter_config.json"), encoding="utf-8") as f:
            r = int(json.load(f).get("r", 8))
        ec.max_loras, ec.max_lora_rank = 1, next((k for k in (8, 16, 32, 64) if k >= r), r)
    t0 = time.perf_counter()
    if args.synthetic:
        from swiftllm_b200.model_config import LLAMA3_8B, LLAMA3_70B
        from swiftllm_b200.worker.weight import synthetic_getter
        mc = swiftllm_b200.LlamaModelConfig(dict(LLAMA3_8B if args.synthetic == "llama3-8b" else LLAMA3_70B))
        model = swiftllm_b200.LlamaModel(ec, mc)
        model.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
        g = torch.Generator().manual_seed(0)
        input_ids = [torch.randint(0, mc.vocab_size, (n,), generator=g).tolist() for n in (9, 5, 1200, 6)]
        show = lambda ids: " ".join(map(str, ids))
    else:
        from transformers import AutoTokenizer
        model = swiftllm_b200.LlamaModel(ec)
        model.load_weights()
        tok = AutoTokenizer.from_pretrained(args.model_path)
        prompts = ["Life blooms like a flower, far away", "one two three four five",
                   "A B C D E F G H I J K L M N O P Q R S T U V", "To be or not to be,"]
        input_ids = tok(prompts)["input_ids"]
        show = lambda ids: tok.decode(ids, skip_special_tokens=True)
    if args.lora:
        model.load_lora(0, args.lora)
    num_blocks = model.profile_num_blocks()
    model.init_kvcache_and_swap(num_blocks)
    if args.lora:
        with_adapter(model, 0)
    print(f"{num_blocks} KV blocks; model ready in {time.perf_counter() - t0:.1f} s")

    params = swiftllm_b200.SamplingParams(args.temperature, top_k=args.top_k, top_p=args.top_p, seed=args.seed, logprobs=args.logprobs,
                                          prompt_logprobs=args.prompt_logprobs,
                                          repetition_penalty=args.repetition_penalty, frequency_penalty=args.frequency_penalty,
                                          presence_penalty=args.presence_penalty)
    if args.temperature == 0 and args.logprobs is None and args.prompt_logprobs is None and not params.has_penalties():
        params = None
    logs = [[] for _ in range(len(input_ids) * args.n)]
    prompt_logs = [[] for _ in input_ids]
    outputs, t_prefill, t_decode = generate(model, input_ids, args.new_tokens, args.chunk, params, logs, args.speculate, args.n,
                                            prompt_logs)
    for i, pls in enumerate(prompt_logs if args.prompt_logprobs is not None else []):
        lp = np.concatenate([pl.logprobs for pl in pls]) if pls else np.zeros((0,))
        ppl = float(np.exp(-lp.astype(np.float64).mean())) if lp.size else float("nan")
        print(f"prompt {i}: {lp.size} scored tokens, perplexity {ppl:.3f}")
        for pl in pls[:1]:
            for j in range(min(4, len(pl.token_ids))):
                top = ", ".join(f"{show([int(t)])!r}:{float(v):.3f}" for t, v in zip(pl.top_ids[j], pl.top_logprobs[j]))
                print(f"    pos {pl.first_position + j} {show([int(pl.token_ids[j])])!r} {pl.logprobs[j]:.4f} "
                      f"rank {pl.ranks[j]}   top [{top}]")
    seq_ids = list(range(len(outputs)))
    # rows of prompt i: i, then its forks
    rows = [k for i in range(len(input_ids)) for k in [i] + [len(input_ids) + i * (args.n - 1) + j for j in range(args.n - 1)]]
    for k in rows:
        p, o, lg = input_ids[k if k < len(input_ids) else (k - len(input_ids)) // (args.n - 1)], outputs[k], logs[k]
        print(f"[{len(p)} prompt tokens] -> {show(o)}")
        for r in lg if args.logprobs is not None else []:      # log-probabilities of the raw model distribution (before penalties, temperature / top-k / top-p)
            top = ", ".join(f"{show([t])!r}:{lp:.3f}" for t, lp in r.top)
            print(f"    {show([r.token])!r} {r.logprob:.4f}   top [{top}]")
    print(f"prefill {t_prefill * 1e3:.1f} ms ({sum(map(len, input_ids)) / t_prefill:.0f} tok/s), "
          f"decode {t_decode / max(1, args.new_tokens - 1) * 1e3:.2f} ms/step")
    model.free_seqs_resources(seq_ids)


if __name__ == "__main__":
    main()
