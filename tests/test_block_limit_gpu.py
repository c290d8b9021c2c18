"""GPU: a decode step whose sequence would need more than max_blocks_per_seq blocks is refused alike on the eager path and on the
CUDA-graph path: the same RuntimeError before anything is enqueued, the block table, free map and host mirror unchanged, and
the next valid step replays the captured graph to the eager path's tokens.  Both paths count a step's blocks with
BlockManager.reserve_blocks_for_seqs; the graph path must not replay a step its allocation kernel would refuse, or the KV
store would index past the sequence's row of the block table."""
import numpy as np
import pytest
import torch

from oracle.model import OracleWeights
from test_model_gpu import TINY2, _make_model

pytestmark = pytest.mark.gpu
BS, MBPS = 16, 4
ENG = dict(block_size=BS, num_cpu_blocks=0, max_seqs_in_block_table=4, max_blocks_per_seq=MBPS, num_blocks=16)


def _state(m):
    torch.cuda.synchronize()
    bm = m.gpu_block_manager
    return (bm.block_table.cpu(), bm.num_seq_allocated_blocks.cpu(), bm.is_block_free.cpu(), bm._host_nsab.copy(),
            bm.num_free_blocks)


def _assert_same(a, b):
    assert torch.equal(a[0], b[0]), "block table changed"
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), "allocation counts or free map changed"
    assert np.array_equal(a[3], b[3]) and a[4] == b[4], "host mirror or free count changed"


def test_step_past_max_blocks_per_seq_is_refused_on_both_paths():
    w = OracleWeights.random(TINY2, dtype=torch.bfloat16, seed=7, std=0.05)
    eager = _make_model(TINY2, ENG, w, dtype="bfloat16", graph=False)
    graph = _make_model(TINY2, ENG, w, dtype="bfloat16", graph=True)
    rng = np.random.default_rng(7)
    prompts = [rng.integers(0, TINY2["vocab_size"], size=n).tolist() for n in (MBPS * BS, 20, 31)]   # sequence 0 fills its row
    sids = [0, 1, 2]
    a = eager.forward(prompts, sids, [])
    assert graph.forward(prompts, sids, []) == a
    lens = [len(p) for p in prompts]

    def decode(batch, ids, step_lens):
        x = eager.forward([[t] for t in ids], batch, step_lens)
        y = graph.forward([[t] for t in ids], batch, step_lens)
        assert x == y, "graph and eager tokens differ"
        assert torch.equal(eager.post_layer.last_logits, graph.post_layer.last_logits)
        return x

    t12 = decode([1, 2], a[1:], [lens[1] + 1, lens[2] + 1])          # captures the graph of batch size 2
    assert len(graph._graphs) == 1
    messages = []
    for m in (eager, graph):
        before = _state(m)
        with pytest.raises(RuntimeError) as e:
            m.forward([[a[0]], [t12[0]]], [0, 1], [lens[0] + 1, lens[1] + 2])     # sequence 0 would need block MBPS + 1
        messages.append(str(e.value))
        _assert_same(_state(m), before)
    assert messages == [f"sequence needs {MBPS + 1} blocks > max_blocks_per_seq={MBPS}"] * 2
    assert len(graph._graphs) == 1

    decode([1, 2], t12, [lens[1] + 2, lens[2] + 2])                   # the same graph; sequence 2 takes a block
    assert len(graph._graphs) == 1
    se, sg = _state(eager), _state(graph)
    n = se[1]
    assert torch.equal(n, sg[1]) and torch.equal(se[2], sg[2]) and np.array_equal(se[3], sg[3]) and se[4] == sg[4]
    for s in sids:
        assert torch.equal(se[0][s, :n[s]], sg[0][s, :n[s]])
    assert torch.equal(eager.k_cache, graph.k_cache) and torch.equal(eager.v_cache, graph.v_cache)
    assert graph.gpu_block_manager.check_device_status() == 1       # the replay allocated it, with no error flag

    # refused alone: the graph of batch size 1 is captured first (its warm-up runs on a scratch cache, the capture executes
    # nothing), then the step is refused with nothing changed and nothing launched on the real tables
    for m in (eager, graph):
        before = _state(m)
        with pytest.raises(RuntimeError, match=f"^sequence needs {MBPS + 1} blocks > max_blocks_per_seq={MBPS}$"):
            m.forward([[a[0]]], [0], [lens[0] + 1])
        _assert_same(_state(m), before)
    assert len(graph._graphs) == 2
    assert graph.gpu_block_manager.check_device_status() == 1
