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
    ... --repetition-penalty 1.1 --frequency-penalty 0.5 --presence-penalty 0.3    discourage repeats (vLLM's definitions)
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import swiftllm_b200  # noqa: E402


def generate(model, input_ids, new_tokens: int, chunk: int = 0, params=None, logs=None):
    """Generation for a batch of prompts (sequence i uses block-table row i), greedy unless `params` (one
    swiftllm_b200.SamplingParams for every sequence) is given.  chunk > 0: the prompts are prefilled `chunk` tokens at a time
    through the paged cache.  Returns (token lists, prefill seconds, decode seconds).
    With params.logprobs set, logs[i] (a list per sequence) receives the TokenLogprobs of every generated token."""
    seq_ids = list(range(len(input_ids)))
    sp = (lambda n: None) if params is None else (lambda n: [params] * n)
    want_lp = params is not None and params.logprobs is not None
    logs = logs if logs is not None else [[] for _ in input_ids]

    def step(*args, **kw):
        if not want_lp:
            return model.forward(*args, **kw)
        return model.forward_with_logprobs(*args, **kw)
    t0 = time.perf_counter()
    if chunk > 0:                      # every call carries the next chunk of each unfinished prompt
        done = [0] * len(input_ids)
        last = [None] * len(input_ids)
        while any(d < len(p) for d, p in zip(done, input_ids)):
            live = [i for i in seq_ids if done[i] < len(input_ids[i])]
            toks = step([input_ids[i][done[i]:done[i] + chunk] for i in live], live, [],
                        prefill_prefix_lens_list=[done[i] for i in live], sampling_params_list=sp(len(live)))
            for i, t in zip(live, toks):
                done[i] = min(len(input_ids[i]), done[i] + chunk)
                if done[i] == len(input_ids[i]):
                    last[i] = t             # the token sampled after the LAST chunk is the first generated token
    else:
        last = step(input_ids, seq_ids, [], sampling_params_list=sp(len(seq_ids)))
    if want_lp:
        for lg, r in zip(logs, last):
            lg.append(r)
        last = [r.token for r in last]
    t_prefill = time.perf_counter() - t0
    outputs = [[t] for t in last]
    seq_lens = [len(p) for p in input_ids]
    t0 = time.perf_counter()
    for _ in range(new_tokens - 1):
        seq_lens = [n + 1 for n in seq_lens]
        last = step([[t] for t in last], seq_ids, seq_lens, sampling_params_list=sp(len(seq_ids)))
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
    ap.add_argument("--repetition-penalty", type=float, default=1.0, help="divide / multiply the logits of seen tokens (1 = off)")
    ap.add_argument("--frequency-penalty", type=float, default=0.0, help="subtract this times each token's output count (0 = off)")
    ap.add_argument("--presence-penalty", type=float, default=0.0, help="subtract this from every token already output (0 = off)")
    args = ap.parse_args()

    ec = swiftllm_b200.EngineConfig(model_path=args.model_path or "", use_dummy=False, block_size=16, gpu_mem_utilization=0.9,
                                    num_cpu_blocks=0, max_seqs_in_block_table=128, max_blocks_per_seq=2048, max_batch_size=16,
                                    max_tokens_in_batch=2048 * 16, dtype=args.dtype, use_cuda_graph=args.cuda_graph)
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
    num_blocks = model.profile_num_blocks()
    model.init_kvcache_and_swap(num_blocks)
    print(f"{num_blocks} KV blocks; model ready in {time.perf_counter() - t0:.1f} s")

    params = swiftllm_b200.SamplingParams(args.temperature, top_k=args.top_k, top_p=args.top_p, seed=args.seed, logprobs=args.logprobs,
                                          repetition_penalty=args.repetition_penalty, frequency_penalty=args.frequency_penalty,
                                          presence_penalty=args.presence_penalty)
    if args.temperature == 0 and args.logprobs is None and not params.has_penalties():
        params = None
    logs = [[] for _ in input_ids]
    outputs, t_prefill, t_decode = generate(model, input_ids, args.new_tokens, args.chunk, params, logs)
    seq_ids = list(range(len(input_ids)))
    for p, o, lg in zip(input_ids, outputs, logs):
        print(f"[{len(p)} prompt tokens] -> {show(o)}")
        for r in lg:      # log-probabilities of the raw model distribution (before penalties, temperature / top-k / top-p)
            top = ", ".join(f"{show([t])!r}:{lp:.3f}" for t, lp in r.top)
            print(f"    {show([r.token])!r} {r.logprob:.4f}   top [{top}]")
    print(f"prefill {t_prefill * 1e3:.1f} ms ({sum(map(len, input_ids)) / t_prefill:.0f} tok/s), "
          f"decode {t_decode / max(1, args.new_tokens - 1) * 1e3:.2f} ms/step")
    model.free_seqs_resources(seq_ids)


if __name__ == "__main__":
    main()
