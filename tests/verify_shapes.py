"""Shapes of the speculative-verification attention tests, shared by the GPU tests (tests/test_speculative_gpu.py,
tests/test_attention_regimes_gpu.py) and the CPU check of their power (tests/test_attention_check_cpu.py), so both run
the same geometries and the same row / prefix layouts."""
import numpy as np
import torch

# (g, nkv, max_rows, wgmma N): every width with a power-of-two and a non-power-of-two group (dead columns between g * max_rows
# and N: 1 for g3 x 5, 8 for g3 x 8), g16 (one kv head fills the box), the shapes the kernel exists for (Llama-3-8B, g4, up
# to 8 rows; g8 up to 4 rows), and past 32 columns the paged-prefill fallback
VERIFY_GEOMS = [(1, 8, 8, 8), (2, 2, 4, 8),
                (4, 4, 4, 16), (3, 1, 5, 16), (16, 1, 1, 16),
                (4, 8, 8, 32), (8, 8, 4, 32), (3, 8, 8, 32), (5, 2, 6, 32), (7, 4, 4, 32), (12, 2, 2, 32), (16, 2, 2, 32),
                (5, 8, 7, None), (8, 4, 5, None), (8, 8, 8, None)]
LAYOUTS = ["short_many", "long_few"]


def verify_np(g, max_rows):
    """wgmma N of the verify kernel for a launch: g * max_rows columns padded to 8, 16 or 32; None past 32 (fallback)."""
    cols = g * max_rows
    return next((n for n in (8, 16, 32) if cols <= n), None)


def geom_id(gm):
    g, nkv, r, npad = gm
    return f"g{g}x{r}-{nkv}kv-" + (f"np{npad}" if npad else f"{g * r}cols")


def verify_layout(layout, g, max_rows):
    """(rows, prefix) of the entries, rows capped at max_rows.
    short_many: 48 entries, ragged rows 1..8, prefixes at page edges and small random ones (one split per item).
    long_few: three long entries (several splits): columns of early rows see nothing of the last split; the second entry
    ends exactly at the last slot of a 256-block table row."""
    if layout == "short_many":
        rows = [1 + i % 8 for i in range(48)]
        prefix = np.random.default_rng(10 * g + max_rows).integers(0, 300, size=48).tolist()
        prefix[:6] = [0, 1, 15, 16, 17, 31]
    else:
        rows, prefix = [8, 5, 1], [3001, 4096 - 5, 17]
    return [min(r, max_rows) for r in rows], prefix


def random_kv_q(gen, nblk, layers, nkv, T, nq, D, bs, dtype):
    """K and V caches [nblk, layers, nkv, bs, D] and packed q [T, nq, D] of randn values, drawn in that order from `gen`."""
    kc = torch.randn(nblk, layers, nkv, bs, D, generator=gen).to(dtype)
    vc = torch.randn(nblk, layers, nkv, bs, D, generator=gen).to(dtype)
    q = torch.randn(T, nq, D, generator=gen).to(dtype)
    return kc, vc, q
