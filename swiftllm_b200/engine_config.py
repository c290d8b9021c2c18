"""Engine configuration.  The first nine fields and their CLI flags are the reference's
(swiftllm/engine_config.py:4-84); the trailing fields (with defaults) are additions for the H100 data plane."""
import argparse
import dataclasses


@dataclasses.dataclass
class EngineConfig:
    # Model loading parameters
    model_path: str
    use_dummy: bool

    # PagedAttention-related parameters
    block_size: int
    gpu_mem_utilization: float
    num_cpu_blocks: int
    max_seqs_in_block_table: int
    max_blocks_per_seq: int

    # Scheduling-related parameters
    max_batch_size: int
    max_tokens_in_batch: int

    # ---- additions ----
    dtype: str = "float16"          # "float16" (the reference's hard-coded dtype) or "bfloat16"
    tp_size: int = 1                # tensor-parallel world size (heads / FFN columns), one process per GPU
    tp_rank: int = 0
    pin_swap_space: bool = True     # the reference's swap space is pageable (model.py:158-159)
    use_cuda_graph: bool = False    # capture pure-decode steps into CUDA graphs
    max_cuda_graphs: int = 16       # decode graphs kept (keyed by batch size x length bucket), least recently used evicted
    # TP exchange: True = one-shot peer-memory all-reduce fused with add+RMSNorm (tp_comm.py), False = NCCL all-reduce +
    # a separate kernel, None = automatic (what was measured fastest: one-shot at tp_size 2 and 4, "two_shot_nvls" at 8 with
    # "two_shot" and then NCCL as fall-backs when multicast / peer memory is unavailable),
    # "two_shot" = the row-owner (reduce-scatter + all-gather) variant of the fused kernel, meant for tp_size 8,
    # "two_shot_nvls" = the same with the reduction and the broadcast done by the NVSwitch (multimem.ld_reduce / multimem.st),
    # "ll" / "ll_nvls" = decode-sized exchanges (<= 1024 rows) through the barrier-free push kernel (csrc/allreduce_ll.cu: data
    # lines carry their own epoch tag; "ll_nvls" broadcasts the normalised rows with one multimem.st), larger ones two-shot
    fused_allreduce: object = None
    # TP: shard lm_head by vocabulary rows (each rank computes logits of V/tp_size tokens; the greedy token is found with one
    # tiny all-gather of per-rank (max logit, argmax) pairs) instead of replicating the 1 GB matrix on every rank.
    # SURVEY.md §8 f-3.  None = automatic: sharded whenever tp_size > 1 and divides the vocabulary.
    shard_lm_head: object = None
    # pure-decode steps: rotary embedding + KV store of the new rows in ONE launch per layer instead of two.
    # Bit-identical to the two kernels (tests/test_decode_fusion_gpu.py); one launch less per layer.
    fuse_rotary_store: bool = True
    # swap in / out with device-resident id lists and one gather/scatter kernel over the pinned, mapped swap space (no host
    # syncs) instead of `.tolist()` + cudaMemcpyAsync per run (SURVEY.md §8 f-4).  Needs pin_swap_space.  Tested by
    # tests/test_swap_device_gpu.py; opt-in: its copy speed (SM loads / stores over PCIe) against the DMA path is unmeasured.
    device_swap: bool = False
    # swap copies run on a dedicated copy stream (SURVEY.md §8 f-4): swap_in_seqs / swap_out_seqs return as soon as the block
    # tables are updated and the copy is enqueued; the next forward waits for it on the device right before its first KV-cache
    # access.  (The wait cannot be later: freed blocks are handed out again lowest-id-first - the reference's order, which the
    # block-index parity depends on - so the next step's KV store may target exactly the blocks being copied out.)
    swap_on_copy_stream: bool = False

    @staticmethod
    def add_cli_args(parser: argparse.ArgumentParser):
        parser.add_argument("--model-path", type=str, required=True,
                            help="Path to the model directory (config.json + safetensors / pytorch_model.bin)")
        parser.add_argument("--use-dummy", action="store_true", help="Use dummy weights (mainly for profiling)")
        parser.add_argument("--block-size", type=int, default=16, help="Block size for PagedAttention")
        parser.add_argument("--gpu-mem-utilization", type=float, default=0.97, help="Fraction of GPU memory to be used")
        parser.add_argument("--num-cpu-blocks", type=int, default=2048, help="Number of CPU blocks")
        parser.add_argument("--max-seqs-in-block-table", type=int, default=4096,
                            help="Maximum number of sequences in the block table")
        parser.add_argument("--max-blocks-per-seq", type=int, default=32768, help="Maximum number of blocks per sequence")
        parser.add_argument("--max-batch-size", type=int, default=512, help="Maximum batch size")
        parser.add_argument("--max-tokens-in-batch", type=int, default=32768, help="Maximum number of tokens in a batch")
        parser.add_argument("--dtype", type=str, default="float16", choices=["float16", "bfloat16"])
        parser.add_argument("--use-cuda-graph", action="store_true")
