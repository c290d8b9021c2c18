// What paged_attn.cu (the C entry points and the split planner) and paged_attn_tc.cu (the generation-2 kernels) share.
#pragma once
#include "common.cuh"

namespace sllm {

// Kernel parameters of paged_attn_tc_kernel (decode).
struct TcParams {
    const int32_t* block_table; const int32_t* seq_ids;
    const int32_t* seq_lens;          // decode only
    void* o; float* part_o; float* part_lse;
    float scale_log2e;
    int split_tokens, num_splits, cur_layer, num_layers, nq, nkv, max_blocks_per_seq;
    // filled by the launcher
    int num_items;
    // shared-memory placement of the 1 KiB atoms of a KV tile and the matching descriptor strides
    int page_stride, half_stride, k_sbo, v_lbo, v_sbo, tma_4d;
};

// Kernel parameters of paged_attn_verify_kernel (speculative verification).  A struct of its own rather than more fields of
// TcParams: with them (and the three tensor maps) the decode kernel's parameters pass 512 bytes, and nvcc 12.9 then compiles
// it to a different instruction stream (about 10 % fewer instructions, 102 instead of 153 registers at NP = 16; not measured).
struct TcVerifyParams : TcParams {
    const int32_t* start_locs; const int32_t* row_counts; const int32_t* prefix_lens;
    int32_t* row_lens;                // when split: visible length of each row, the merge kernel's seq_lens
    int qrows;                        // rows of the Q box (the largest row count of the batch)
};

// One launch: the caller fills everything but the launcher's part of `p`.  `split_tokens` / `num_splits` come from the
// planner in paged_attn.cu, which also merges the partials.
struct TcLaunch {
    TcVerifyParams p;                 // decode uses the TcParams part
    const void* q; const void* k_cache; const void* v_cache;
    int64_t num_blocks, q_row_stride;
    int64_t num_tokens;               // rows of q and o (decode: one per sequence)
    int num_seqs;                     // sequences (decode) / entries (verify)
    sllm_dtype_t dtype;
    int num_sms;
    cudaStream_t stream;
};

bool tc_paged_supported(int head_dim, int block_size, int nq, int nkv, int64_t num_blocks, int num_layers);
bool tc_verify_supported(int head_dim, int block_size, int nq, int nkv, int max_rows, int64_t num_blocks, int num_layers,
                         int64_t num_tokens);
// Launch the persistent kernel; return 0 / error like the C entry points.
int launch_paged_tc(const TcLaunch& a);
int launch_paged_verify_tc(const TcLaunch& a);

}  // namespace sllm
