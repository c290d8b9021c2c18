// Repetition / frequency / presence penalties applied in place to [rows, V] 16-bit logits, with the token history read from
// the device-resident token pages (token_cache int32 [num_blocks, block_size], addressed through the block table like a KV page;
// each entry is id | is_output << 31).
// Semantics (restated in numpy by tests/penalties_oracle.py), per row with r, f, p its penalties and the history = positions
// [0, pos) of its sequence (pages for [0, pos - n_new), this step's n_new input tokens for the rest):
//   c_out(v)  number of output tokens equal to v; seen(v): v occurs among the prompt or output tokens;
//   seen v    l = float(logit); l = l > 0 ? l / r : l * r; t = f * float(c_out); t = t + p if c_out > 0; l = l - t; stored
//             rounded once to the storage dtype (round to nearest even).  fp32, IEEE, no contraction;
//   other v   the entry keeps its bits.
// Ids outside [vocab_offset, vocab_offset + vocab_size) are not this launch's (absent); an invalid id or block id in the history
// is skipped, never dereferenced.  Rows with r == 1, f == 0, p == 0 are skipped entirely (nothing read, recorded or modified).
// After counting, the row's new tokens are written to positions [pos - n_new, pos) of its pages - disjoint from what is read.
//
// Layout: one thread-block cluster of C CTAs per penalised row, with the cluster geometry (4 bytes per entry) and launch of
// vocab_select.cuh.  The cluster keeps a u32 slot per vocabulary id of the launch's shard in distributed shared memory, CTA k
// owning ids [k * slice, (k + 1) * slice): bit 31 = seen in the prompt, the low bits
// count output tokens (exact up to 2^31 - 1).  Every CTA counts a strided share of the history into whichever CTA owns each id;
// lanes of a warp holding the same (id, kind) are merged first (__match_any_sync), so one id repeated thousands of times costs one
// DSMEM atomic per warp, not one per occurrence.  After a cluster barrier each CTA rewrites the entries of its slice whose slot
// is non-zero.  Counts are integers: the result does not depend on the order of the atomics, the cluster size or the batch.
// Algorithmic bytes per penalised row: 4 * pos (history) + 4 * n_new (pages written) + 4 * distinct ids (logits read / written).
//
// N-gram controls (the kNgram instantiation, sllm_apply_penalties_ngram; restated by tests/ngram_oracle.py).  With x[0, L) the
// history above (L = pos; ids compared without the output bit; an unmapped position or invalid block id matches nothing):
//   m(j)  the largest m in [0, min(j, 50)] with x[j - k] == x[L - k] for k = 1 .. m;  M(v) = max m(j) over the j with x[j] == v;
//   ban   (no_repeat_ngram_size n >= 1) l = -inf where M(v) >= n - 1 (Hugging Face's no_repeat_ngram_size);
//   DRY   (dry_multiplier > 0) with b the smallest k >= 1 such that x[L - k] is one of the row's 16 breaker ids (51 if none of
//         the last 50 is) and D(v) = min(M(v), b - 1) for a v that is no breaker: where D >= A (dry_allowed_length),
//         q = multiplier, D - A times q = q * base, l = l - q (fp32, round to nearest; text-generation-webui's DRY).
// Per entry: l = float(logit), the penalties above when the row has any, DRY, the ban, one rounding; an entry none of them
// touches keeps its bits.  Layout: the cluster also keeps a u32 match slot per id (M + 1, 0 = none), so 8 bytes per entry.
// Each CTA walks its strided share of the history in tiles of kThreads positions, staged in shared memory with the kMaxMatch
// positions before them; the row's last kMaxMatch tokens are staged once.  A position whose m(j) reaches the row's smallest
// active threshold (n - 1, A) takes the max over the warp's lanes with the same id (__match_any_sync + __reduce_max_sync) and
// one DSMEM atomicMax into the owning slot.  M is an integer maximum: the result does not depend on atomic order, cluster
// size, batch or shard.  A launch without these controls runs the plain instantiation (4-byte slots) unchanged.
#include "vocab_select.cuh"

namespace sllm {
namespace {

constexpr uint32_t kOutputBit = 0x80000000u;       // token page word: id | kOutputBit for an output token
constexpr uint32_t kSeenInPrompt = 0x80000000u;    // cluster slot: set when the id occurs among the prompt tokens
constexpr uint32_t kAbsentId = 0x7fffffffu;        // recorded for a negative input id: >= vocab_offset + vocab_size always

constexpr int kSlotBytes = 4, kSlotAlign = 4;     // cluster slots: uint32, slices zeroed as whole uint4 vectors
constexpr int kNgramSlotBytes = 8;                 // kNgram: a count slot and a match slot per id
constexpr int kMaxMatch = 50;                      // longest match m(j) (text-generation-webui's cap)
constexpr int kMaxBreakers = 16;                   // DRY sequence breakers per row (-1: unused)
constexpr uint32_t kTileNone = 0x80000000u, kTailNone = 0x80000001u;   // staged unmapped positions: never equal to each other
                                                                       // or to an id (ids < 2^31)
// shared memory of the kNgram instantiation after its two slot arrays: the tile with its kMaxMatch positions before it, the
// row's last kMaxMatch tokens, and the breaker distance b
constexpr int kNgramStageWords = kThreads + kMaxMatch + 64;

// Per-row device arrays of the n-gram controls (nullptr members: the plain instantiation)
struct NgramRows {
    const int32_t* no_repeat;       // n, 0: no ban
    const int32_t* allowed;         // A
    const float* multiplier;        // 0: no DRY
    const float* base;
    const int32_t* breakers;        // [rows, kMaxBreakers] global ids, -1 unused
};

template <typename T, bool kNgram>
__global__ void __launch_bounds__(kThreads) penalty_kernel(
    T* __restrict__ logits, int64_t row_stride, int V, int64_t vocab_offset, int slice, const float* __restrict__ rep,
    const float* __restrict__ freq, const float* __restrict__ pres, const int32_t* __restrict__ seq_ids,
    const int32_t* __restrict__ pos, const int32_t* __restrict__ input_ids, const int32_t* __restrict__ last_token_indices,
    const int32_t* __restrict__ prefill_seq_lens, int num_prefill_rows, const int32_t* __restrict__ block_table,
    int block_table_stride, int block_size, int32_t* token_cache, int64_t num_blocks, NgramRows ng) {
    extern __shared__ uint32_t slots[];

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned C = cluster.num_blocks(), rank = cluster.block_rank();
    const int64_t row = blockIdx.x / C;
    const float r = rep[row], f = freq[row], p = pres[row];
    if constexpr (!kNgram) {
        if (r == 1.f && f == 0.f && p == 0.f) return;                 // the whole cluster leaves, before any DSMEM access
    }
    const bool penalised = !(r == 1.f && f == 0.f && p == 0.f);
    int ban = 0, allowed = 0;
    float mult = 0.f, base = 1.f;
    if constexpr (kNgram) {
        ban = ng.no_repeat[row];
        allowed = max(0, ng.allowed[row]);
        mult = ng.multiplier[row];
        base = ng.base[row];
        if (!penalised && ban <= 0 && !(mult > 0.f)) return;       // the whole cluster leaves, before any DSMEM access
    }
    const bool dry = mult > 0.f;
    // matches shorter than the smallest active threshold change nothing: they are not merged
    const int thr = min(ban > 0 ? ban - 1 : INT_MAX, dry ? allowed : INT_MAX);
    uint32_t* match = slots + slice;                                   // kNgram: M + 1 per id of the slice, 0 = none
    uint32_t* tile = match + slice;                                    // kNgram: positions [t0 - kMaxMatch, t0 + kThreads)
    uint32_t* tail = tile + kThreads + kMaxMatch;                      // kNgram: positions [L - kMaxMatch, L)
    int* brk_dist = reinterpret_cast<int*>(tail + kMaxMatch);          // kNgram: b

    const int begin = (int)rank * slice;
    const int n = max(0, min(V, begin + slice) - begin);
    for (int i = 4 * threadIdx.x; i < (kNgram ? 2 : 1) * slice; i += 4 * blockDim.x)
        *reinterpret_cast<uint4*>(slots + i) = make_uint4(0, 0, 0, 0);

    // ---- the row's history: positions [0, hist) from the pages, then its n_new input tokens
    const int P = pos[row];
    const bool prefill = row < num_prefill_rows;
    const int n_new = max(0, prefill ? prefill_seq_lens[row] : 1);
    const int64_t first_in = (int64_t)last_token_indices[row] - n_new + 1;
    const uint32_t new_flag = prefill ? 0u : kOutputBit;
    auto new_word = [&](int j) -> uint32_t {                         // page word of the row's j-th new token
        const int32_t id = input_ids[first_in + j];
        return (id >= 0 ? (uint32_t)id : kAbsentId) | new_flag;
    };
    const int hist = max(0, P - n_new);
    const int max_pos = block_table_stride * block_size;             // positions the block-table row can address
    const int32_t* bt = block_table + (int64_t)seq_ids[row] * block_table_stride;
    auto page_slot = [&](int q) -> int64_t {                          // index into token_cache of position q, -1 if unmapped
        if (q < 0 || q >= max_pos) return -1;
        const int64_t b = bt[q / block_size];
        return (b >= 0 && b < num_blocks) ? b * block_size + q % block_size : -1;
    };
    cluster.sync();                                                   // every slot zeroed before any CTA adds to it

    const int total = hist + n_new;
    const int lane = threadIdx.x & 31;
    // counts one (word, valid) of a warp's lanes into the owning slots
    auto count = [&](uint32_t word, bool valid) {
        const bool is_out = (word & kOutputBit) != 0;
        const int64_t local = (int64_t)(word & ~kOutputBit) - vocab_offset;
        valid = valid && local >= 0 && local < V;
        const unsigned long long key = valid ? ((unsigned long long)local << 1) | (is_out ? 1ull : 0ull) : ~0ull;
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        if (valid && lane == __ffs(peers) - 1) {
            uint32_t* dst = cluster.map_shared_rank(slots, (unsigned)(local / slice)) + (local % slice);
            if (is_out) atomicAdd(dst, (uint32_t)__popc(peers));
            else atomicOr(dst, kSeenInPrompt);
        }
    };
    if constexpr (!kNgram) {
        for (int i0 = (int)(rank * blockDim.x + (threadIdx.x & ~31)); i0 < total; i0 += (int)(C * blockDim.x)) {
            const int i = i0 + lane;
            uint32_t word = 0;
            bool valid = false;
            if (i < hist) {
                const int64_t s = page_slot(i);
                if (s >= 0) { word = (uint32_t)token_cache[s]; valid = true; }
            } else if (i < total) {
                word = new_word(i - hist);
                valid = true;
            }
            count(word, valid);
        }
    } else {
        // the word at position q and whether it is mapped
        auto word_at = [&](int q, uint32_t& word) -> bool {
            if (q < 0 || q >= total) return false;
            if (q < hist) {
                const int64_t s = page_slot(q);
                if (s < 0) return false;
                word = (uint32_t)token_cache[s];
                return true;
            }
            word = new_word(q - hist);
            return true;
        };
        if (threadIdx.x < kMaxMatch) {
            uint32_t w = 0;
            tail[threadIdx.x] = word_at(total - kMaxMatch + (int)threadIdx.x, w) ? (w & ~kOutputBit) : kTailNone;
        }
        if (threadIdx.x == 0) *brk_dist = kMaxMatch + 1;
        __syncthreads();
        if (dry && threadIdx.x < kMaxMatch) {                         // b: the nearest breaker among the last kMaxMatch tokens
            const uint32_t t = tail[kMaxMatch - 1 - threadIdx.x];
            bool is_brk = false;
            for (int k = 0; k < kMaxBreakers; k++) is_brk |= (int64_t)ng.breakers[row * kMaxBreakers + k] == (int64_t)t;
            if (is_brk) atomicMin(brk_dist, (int)threadIdx.x + 1);
        }
        for (int t0 = (int)(rank * blockDim.x); t0 < total; t0 += (int)(C * blockDim.x)) {       // block-uniform
            const int i = t0 + (int)threadIdx.x;
            uint32_t word = 0;
            const bool valid = word_at(i, word);
            __syncthreads();                                           // the previous tile has been read
            tile[kMaxMatch + threadIdx.x] = valid ? (word & ~kOutputBit) : kTileNone;
            if (threadIdx.x < kMaxMatch) {
                uint32_t w = 0;
                const int q = t0 - kMaxMatch + (int)threadIdx.x;
                tile[threadIdx.x] = word_at(q, w) ? (w & ~kOutputBit) : kTileNone;
            }
            __syncthreads();
            if (penalised) count(word, valid);
            // m(i), merged into the owning match slot when it reaches thr
            const int64_t local = (int64_t)(word & ~kOutputBit) - vocab_offset;
            int m = 0;
            const int lim = min(i, kMaxMatch);
            const bool want = valid && local >= 0 && local < V && thr <= lim;
            if (want)
                while (m < lim && tile[kMaxMatch + threadIdx.x - 1 - m] == tail[kMaxMatch - 1 - m]) m++;
            const bool hit = want && m >= thr;
            const unsigned peers = __match_any_sync(0xffffffffu, hit ? (uint32_t)local : 0xffffffffu);
            const unsigned best = __reduce_max_sync(peers, hit ? (unsigned)m + 1u : 0u);
            if (hit && lane == __ffs(peers) - 1)
                atomicMax(cluster.map_shared_rank(match, (unsigned)(local / slice)) + (local % slice), best);
        }
    }
    cluster.sync();                                                   // all counts in place

    // ---- rewrite the seen entries of this CTA's slice
    T* dst = logits + row * row_stride + begin;
    if constexpr (!kNgram) {
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const uint32_t c = slots[j];
            if (c == 0) continue;
            const uint32_t c_out = c & ~kSeenInPrompt;
            float l = Traits<T>::to_f(dst[j]);
            l = l > 0.f ? __fdiv_rn(l, r) : __fmul_rn(l, r);
            float t = __fmul_rn(f, __uint2float_rn(c_out));
            if (c_out > 0) t = __fadd_rn(t, p);
            dst[j] = Traits<T>::from_f(__fsub_rn(l, t));
        }
    } else {
        const int b = *brk_dist;
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const uint32_t c = slots[j], mm = match[j];
            if (c == 0 && mm == 0) continue;
            float l = Traits<T>::to_f(dst[j]);
            bool touched = false;
            if (penalised && c != 0) {
                const uint32_t c_out = c & ~kSeenInPrompt;
                l = l > 0.f ? __fdiv_rn(l, r) : __fmul_rn(l, r);
                float t = __fmul_rn(f, __uint2float_rn(c_out));
                if (c_out > 0) t = __fadd_rn(t, p);
                l = __fsub_rn(l, t);
                touched = true;
            }
            if (mm != 0) {
                const int M = (int)mm - 1;
                if (dry) {
                    const int64_t v = vocab_offset + begin + j;
                    bool is_brk = false;
                    for (int k = 0; k < kMaxBreakers; k++) is_brk |= ng.breakers[row * kMaxBreakers + k] == v;
                    const int D = min(M, b - 1);
                    if (!is_brk && D >= allowed) {
                        float q = mult;
                        for (int k = allowed; k < D; k++) q = __fmul_rn(q, base);
                        l = __fsub_rn(l, q);
                        touched = true;
                    }
                }
                if (ban > 0 && M >= ban - 1) {
                    l = -INFINITY;
                    touched = true;
                }
            }
            if (touched) dst[j] = Traits<T>::from_f(l);
        }
    }

    // ---- record this step's tokens at positions [P - n_new, P)
    for (int j = (int)(rank * blockDim.x + threadIdx.x); j < n_new; j += (int)(C * blockDim.x)) {
        const int64_t s = page_slot(P - n_new + j);
        if (s >= 0) token_cache[s] = (int32_t)new_word(j);
    }
    // no DSMEM access after the last barrier: peers may leave
}

}  // namespace
}  // namespace sllm

namespace sllm {
namespace {

// The kNgram instantiation's geometry: the cluster geometry of 8-byte slots, and the dynamic shared memory of a slice
inline bool ngram_fits(int V) { return slice_fits(V, kMaxCluster, kNgramSlotBytes, kSlotAlign); }
inline ClusterGeometry ngram_geometry(int64_t rows, int V) { return cluster_geometry(rows, V, kNgramSlotBytes, kSlotAlign); }
inline size_t ngram_smem_bytes(int slice) { return (size_t)slice * kNgramSlotBytes + kNgramStageWords * sizeof(uint32_t); }

// The argument checks and the launch of both entry points; ng.no_repeat != nullptr selects the kNgram instantiation.
int apply_penalties(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride, int64_t vocab_offset,
                    const float* repetition_penalty, const float* frequency_penalty, const float* presence_penalty,
                    const int32_t* seq_ids, const int32_t* pos, const int32_t* input_ids, const int32_t* last_token_indices,
                    const int32_t* prefill_seq_lens, int num_prefill_rows, const int32_t* block_table, int block_table_stride,
                    int block_size, int32_t* token_cache, int64_t num_blocks, NgramRows ng, sllm_dtype_t dtype,
                    sllm_stream_t stream, const char* name) {
    const bool ngram = ng.no_repeat != nullptr;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "%s: unsupported dtype tag %d", name, (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= (1 << 20), "%s: num_rows %lld out of range", name, (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "%s: vocab_size must be positive, got %d", name, vocab_size);
    SLLM_REQUIRE(ngram ? ngram_fits(vocab_size) : slice_fits(vocab_size, kMaxCluster, kSlotBytes, kSlotAlign),
                 "%s: vocab_size %d does not fit the shared memory of a %d-CTA cluster", name, vocab_size, kMaxCluster);
    SLLM_REQUIRE(vocab_offset >= 0 && vocab_offset + vocab_size <= (int64_t)INT32_MAX,
                 "%s: global vocabulary indices must stay below 2^31 (vocab_offset %lld)", name, (long long)vocab_offset);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "%s: logits_row_stride %lld < vocab_size %d", name,
                 (long long)logits_row_stride, vocab_size);
    SLLM_REQUIRE(block_size > 0 && block_size <= (1 << 16), "%s: block_size %d out of range", name, block_size);
    SLLM_REQUIRE(block_table_stride > 0 && (int64_t)block_table_stride * block_size <= INT32_MAX,
                 "%s: block_table_stride %d out of range", name, block_table_stride);
    SLLM_REQUIRE(num_blocks >= 0, "%s: num_blocks %lld < 0", name, (long long)num_blocks);
    SLLM_REQUIRE(num_prefill_rows >= 0 && num_prefill_rows <= num_rows, "%s: num_prefill_rows %d out of range", name,
                 num_prefill_rows);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && repetition_penalty && frequency_penalty && presence_penalty && seq_ids && pos && input_ids &&
                 last_token_indices && block_table && token_cache && (num_prefill_rows == 0 || prefill_seq_lens),
                 "%s: null pointer", name);
    SLLM_REQUIRE(!ngram || (ng.allowed && ng.multiplier && ng.base && ng.breakers), "%s: null pointer", name);
    const ClusterGeometry g = ngram ? ngram_geometry(num_rows, vocab_size)
                                    : cluster_geometry(num_rows, vocab_size, kSlotBytes, kSlotAlign);
    if (!ngram)
        SLLM_DISPATCH_DTYPE(dtype, return launch_cluster<penalty_kernel<T, false>>(
                                       num_rows, g.C, (size_t)g.slice * kSlotBytes, (cudaStream_t)stream, name,
                                       (T*)logits, logits_row_stride, vocab_size, vocab_offset, g.slice, repetition_penalty,
                                       frequency_penalty, presence_penalty, seq_ids, pos, input_ids, last_token_indices,
                                       prefill_seq_lens, num_prefill_rows, block_table, block_table_stride, block_size,
                                       token_cache, num_blocks, ng));
    SLLM_DISPATCH_DTYPE(dtype, return launch_cluster<penalty_kernel<T, true>>(
                                   num_rows, g.C, ngram_smem_bytes(g.slice), (cudaStream_t)stream, name, (T*)logits, logits_row_stride, vocab_size, vocab_offset, g.slice,
                                   repetition_penalty, frequency_penalty, presence_penalty, seq_ids, pos, input_ids,
                                   last_token_indices, prefill_seq_lens, num_prefill_rows, block_table, block_table_stride,
                                   block_size, token_cache, num_blocks, ng));
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_apply_penalties(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                    int64_t vocab_offset, const float* repetition_penalty, const float* frequency_penalty,
                                    const float* presence_penalty, const int32_t* seq_ids, const int32_t* pos,
                                    const int32_t* input_ids, const int32_t* last_token_indices,
                                    const int32_t* prefill_seq_lens, int num_prefill_rows, const int32_t* block_table,
                                    int block_table_stride, int block_size, int32_t* token_cache, int64_t num_blocks,
                                    sllm_dtype_t dtype, sllm_stream_t stream) {
    return sllm::apply_penalties(logits, num_rows, vocab_size, logits_row_stride, vocab_offset, repetition_penalty,
                                 frequency_penalty, presence_penalty, seq_ids, pos, input_ids, last_token_indices,
                                 prefill_seq_lens, num_prefill_rows, block_table, block_table_stride, block_size, token_cache,
                                 num_blocks, sllm::NgramRows{}, dtype, stream, "apply_penalties");
}

extern "C" int sllm_apply_penalties_ngram(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                          int64_t vocab_offset, const float* repetition_penalty,
                                          const float* frequency_penalty, const float* presence_penalty,
                                          const int32_t* seq_ids, const int32_t* pos, const int32_t* input_ids,
                                          const int32_t* last_token_indices, const int32_t* prefill_seq_lens,
                                          int num_prefill_rows, const int32_t* block_table, int block_table_stride,
                                          int block_size, int32_t* token_cache, int64_t num_blocks,
                                          const int32_t* no_repeat_ngram_size, const int32_t* dry_allowed_length,
                                          const float* dry_multiplier, const float* dry_base, const int32_t* dry_breakers,
                                          sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(no_repeat_ngram_size, "apply_penalties_ngram: null pointer");
    return sllm::apply_penalties(logits, num_rows, vocab_size, logits_row_stride, vocab_offset, repetition_penalty,
                                 frequency_penalty, presence_penalty, seq_ids, pos, input_ids, last_token_indices,
                                 prefill_seq_lens, num_prefill_rows, block_table, block_table_stride, block_size, token_cache,
                                 num_blocks,
                                 sllm::NgramRows{no_repeat_ngram_size, dry_allowed_length, dry_multiplier, dry_base,
                                                 dry_breakers},
                                 dtype, stream, "apply_penalties_ngram");
}
