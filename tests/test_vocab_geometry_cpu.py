"""CPU: tests/vocab_geometry.py against the sources it restates (csrc/vocab_select.cuh, sampling.cu, logprobs.cu, penalties.cu,
prompt_logprobs.cu), and the table of which batch runs which cluster size at each vocabulary tests/test_vocab_rows_gpu.py uses.
The GPU tests name their cases by the cluster size the mirror gives, so this keeps those names true without a GPU."""
import os
import re
import shutil

import pytest

import vocab_geometry as VG

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swiftllm_b200", "csrc")


def _int_expr(s: str) -> int:
    assert re.fullmatch(r"[\d\s*]+", s), s
    out = 1
    for f in s.split("*"):
        out *= int(f)
    return out


def _one(pattern: str, text: str, what: str) -> str:
    found = re.findall(pattern, text)
    assert len(found) == 1, f"{what}: expected one match of {pattern!r}, found {len(found)}"
    return found[0]


def source_constants(csrc: str) -> dict:
    """The geometry constants as the sources state them."""
    read = lambda f: open(os.path.join(csrc, f)).read()
    vs = read("vocab_select.cuh")
    c = {
        "MAX_CLUSTER": _int_expr(_one(r"constexpr int kMaxCluster = ([\d\s*]+);", vs, "kMaxCluster")),
        "MAX_SLICE_BYTES": _int_expr(_one(r"constexpr int kMaxSliceBytes = ([\d\s*]+);", vs, "kMaxSliceBytes")),
        "SM_TARGET": int(_one(r"while \(c < kMaxCluster && rows \* c \* 2 <= (\d+)\) c \*= 2;", vs, "cluster_geometry")),
        "KEYS": tuple(int(x) for x in _one(r"constexpr int kKeyBytes = (\d+), kKeyAlign = (\d+);", vs, "kKeyBytes")),
        "slice_of": _one(r"inline int64_t slice_of\(int64_t V, int c, int align\) \{ return (.*?); \}", vs, "slice_of"),
        "fit_loop": _one(r"while \(c < kMaxCluster && (!slice_fits\(V, c, bytes_per_entry, align\))\) c \*= 2;", vs, "fit loop"),
    }
    pen = read("penalties.cu")
    c["SLOTS"] = tuple(int(x) for x in _one(r"constexpr int kSlotBytes = (\d+), kSlotAlign = (\d+);", pen, "kSlotBytes"))
    # each cluster kernel sizes its slice, checks the largest V and launches with the same (bytes, align) pair
    for kernel, f, pair in (("sampling", "sampling.cu", "kKeyBytes, kKeyAlign"), ("logprobs", "logprobs.cu", "kKeyBytes, kKeyAlign"),
                            ("penalties", "penalties.cu", "kSlotBytes, kSlotAlign")):
        src = read(f)
        geo = _one(r"cluster_geometry\(num_rows, vocab_size, (\w+, \w+)\)", src, f + " cluster_geometry")
        fit = _one(r"slice_fits\(vocab_size, kMaxCluster, (\w+, \w+)\)", src, f + " slice_fits")
        smem = _one(r"\(size_t\)g\.slice \* (\w+)", src, f + " dynamic shared memory")
        assert geo == fit == pair and smem == pair.split(",")[0], (f, geo, fit, smem)
        c["ENTRY_" + kernel] = c["KEYS"] if pair.startswith("kKey") else c["SLOTS"]
    pl = read("prompt_logprobs.cu")
    c["STAGE_KEYS"] = _int_expr(_one(r"constexpr int kStageKeys = ([\d\s*]+);", pl, "kStageKeys"))
    c["MAX_CAND"] = _int_expr(_one(r"constexpr int kMaxCand = ([\d\s*]+);", pl, "kMaxCand"))
    return c


def mismatches(c: dict) -> list:
    want = {"MAX_CLUSTER": VG.MAX_CLUSTER, "MAX_SLICE_BYTES": VG.MAX_SLICE_BYTES, "SM_TARGET": VG.SM_TARGET, "KEYS": VG.KEYS,
            "SLOTS": VG.SLOTS, "STAGE_KEYS": VG.STAGE_KEYS, "MAX_CAND": VG.MAX_CAND,
            "slice_of": "((V + c - 1) / c + align - 1) / align * align",
            "fit_loop": "!slice_fits(V, c, bytes_per_entry, align)"}
    want.update({"ENTRY_" + k: v for k, v in VG.ENTRY.items()})
    return [(k, c.get(k), v) for k, v in want.items() if c.get(k) != v]


def test_the_mirror_states_the_sources_constants():
    assert mismatches(source_constants(CSRC)) == []


@pytest.mark.parametrize("edit", [("vocab_select.cuh", "kMaxSliceBytes = 200 * 1024", "kMaxSliceBytes = 192 * 1024"),
                                  ("vocab_select.cuh", "rows * c * 2 <= 132", "rows * c * 2 <= 114"),
                                  ("vocab_select.cuh", "kKeyBytes = 2, kKeyAlign = 8", "kKeyBytes = 2, kKeyAlign = 16"),
                                  ("penalties.cu", "kSlotBytes = 4, kSlotAlign = 4", "kSlotBytes = 4, kSlotAlign = 8"),
                                  ("prompt_logprobs.cu", "kStageKeys = 48 * 1024", "kStageKeys = 40 * 1024")],
                         ids=["kMaxSliceBytes", "sm-target", "key-align", "slot-align", "kStageKeys"])
def test_a_changed_source_constant_is_noticed(tmp_path, edit):
    f, old, new = edit
    for name in os.listdir(CSRC):
        if name.endswith((".cu", ".cuh")):
            shutil.copy(os.path.join(CSRC, name), tmp_path / name)
    text = (tmp_path / f).read_text()
    assert old in text
    (tmp_path / f).write_text(text.replace(old, new))
    assert mismatches(source_constants(str(tmp_path))) != []


# The cluster size each batch size runs at each vocabulary of tests/test_vocab_rows_gpu.py: {V: {batch: C}} for 2-byte keys
# (sampling, token logprobs) and 4-byte slots (penalties).  The GPU test ids (C4-V128256, ...) come from the mirror; this table
# pins the mirror.
KEY_TABLE = {
    1000: {1: 8, 3: 8, 16: 8, 17: 4, 24: 4, 33: 4, 34: 2, 40: 2, 66: 2, 67: 1},
    32001: {1: 8, 3: 8, 24: 4, 40: 2, 67: 1},
    128256: {1: 8, 3: 8, 16: 8, 17: 4, 24: 4, 33: 4, 34: 2, 40: 2, 67: 2, 257: 2},
    151936: {1: 8, 3: 8, 24: 4, 40: 2, 67: 2},
    102400: {1: 8, 67: 1}, 102401: {1: 8, 67: 2},
    204800: {1: 8, 67: 2}, 204801: {1: 8, 24: 4, 67: 4},
    409600: {1: 8, 67: 4}, 409601: {1: 8, 67: 8},
    819200: {1: 8, 67: 8},
    1: {1: 8}, 9: {1: 8}, 65: {1: 8},
}
SLOT_TABLE = {
    1000: {1: 8, 3: 8, 24: 4, 40: 2, 67: 1},
    32001: {1: 8, 3: 8, 24: 4, 40: 2, 67: 1},
    128256: {1: 8, 3: 8, 24: 4, 40: 4, 67: 4},
    151936: {1: 8, 3: 8, 24: 4, 40: 4, 67: 4},
    51200: {1: 8, 67: 1}, 51201: {1: 8, 67: 2},
    102400: {1: 8, 67: 2}, 102401: {1: 8, 24: 4, 67: 4},
    204800: {1: 8, 67: 4}, 204801: {1: 8, 67: 8},
    409600: {1: 8, 67: 8},
}


@pytest.mark.parametrize("entry,table", [(VG.KEYS, KEY_TABLE), (VG.SLOTS, SLOT_TABLE)], ids=["keys", "slots"])
def test_which_batch_runs_which_cluster_size(entry, table):
    for V, by_batch in table.items():
        for b, C in by_batch.items():
            assert VG.cluster_geometry(b, V, *entry)[0] == C, (V, b)
        assert VG.accepted(V, *entry)


def test_slices_and_the_largest_vocabularies():
    # the full 200 KB slice at the largest accepted V, and the first V past it refused
    assert VG.cluster_geometry(1, 819200, *VG.KEYS) == (8, 102400) and 102400 * 2 == VG.MAX_SLICE_BYTES
    assert VG.cluster_geometry(1, 409600, *VG.SLOTS) == (8, 51200) and 51200 * 4 == VG.MAX_SLICE_BYTES
    assert not VG.accepted(819201, *VG.KEYS) and not VG.accepted(409601, *VG.SLOTS)
    # each point where the smallest cluster changes
    for V, C in ((102400, 1), (102401, 2), (204800, 2), (204801, 4), (409600, 4), (409601, 8)):
        assert VG.smallest_cluster(V, *VG.KEYS) == C, V
    for V, C in ((51200, 1), (51201, 2), (102400, 2), (102401, 4), (204800, 4), (204801, 8)):
        assert VG.smallest_cluster(V, *VG.SLOTS) == C, V
    # small rows leave whole CTAs of a one-row cluster empty
    assert [e - b for b, e in VG.cta_ranges(9, 8, 8)] == [8, 1, 0, 0, 0, 0, 0, 0]
    assert [e - b for b, e in VG.cta_ranges(65, 8, 8)] == [16, 16, 16, 16, 1, 0, 0, 0]
    # the proposed batches run every cluster size where the slice allows it
    assert [VG.batch_for(C, 128256, *VG.KEYS) for C in (8, 4, 2, 1)] == [12, 24, 40, None]
    assert [VG.batch_for(C, 32001, *VG.KEYS) for C in (8, 4, 2, 1)] == [12, 24, 40, 67]
