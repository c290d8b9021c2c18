"""CPU: tests/row_geometry.py against the launcher it restates (csrc/elementwise.cu: launch_rmsnorm, csrc/common.cuh:
row_threads), the width table tests/test_row_kernels_gpu.py runs, and the fp64 bounds
of tests/row_oracle.py: they accept the kernels' fp32 arithmetic in their own order and in numpy's, and the GPU tests' data
rejects plausible wrong variants of it."""
import os
import re
import shutil

import numpy as np
import pytest
import torch

import kv_geometry as KG
import row_geometry as RG
import row_oracle as RO

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swiftllm_b200", "csrc")
DTYPES = [torch.float16, torch.bfloat16]
ROW_THREADS = ("const int threads = nvec >= 512 ? 512 : (nvec >= 256 ? 256 : ((nvec + 31) / 32) * 32); "
               "return threads < 32 ? 32 : threads;")


def _one(pattern: str, text: str, what: str):
    found = re.findall(pattern, text, re.S)
    assert len(found) == 1, f"{what}: expected one match of {pattern!r}, found {len(found)}"
    return found[0]


def launcher_rules(src: str) -> list:
    """[(condition, vpt, threads expression)] of launch_rmsnorm's register instances, in order, after checking that its generic
    instance stages nvec vectors on row_threads(nvec) threads and fits its shared-memory limit to them first."""
    rules = re.findall(r"if \((nvec [^{]*?)\) \{\s*rmsnorm_kernel<T, FUSED, (\d), QUANT><<<\(unsigned\)T_, (nvec / \d), 0, stream>>>",
                       src)
    _one(r"const int threads = row_threads\(nvec\);\s*const size_t smem = \(size_t\)nvec \* sizeof\(uint4\);\s*"
         r"if \(int e = fit_dynamic_smem<rmsnorm_kernel<T, FUSED, 0, QUANT>>\(smem, what\)\) return e;\s*"
         r"rmsnorm_kernel<T, FUSED, 0, QUANT><<<\(unsigned\)T_, threads, smem, stream>>>", src, "launch_rmsnorm generic")
    return rules


def mismatches(csrc: str) -> list:
    read = lambda f: open(os.path.join(csrc, f)).read()
    try:
        a = launcher_rules(read("elementwise.cu"))
    except AssertionError as e:          # a launch statement the patterns no longer find
        return [str(e)]
    bad = []
    if [(v, t) for _, v, t in a] != [("4", "nvec / 4"), ("2", "nvec / 2")]:
        bad.append(("instances", a))
    # the sources' own conditions pick the instance the mirror picks, at every width the C ABI takes
    for H in range(8, (1 << 16) + 1, 8):
        vpt = next((int(v) for cond, v, _ in a
                    if eval(cond.replace("&&", " and ").replace("/", "//"), {"nvec": H // 8})), 0)
        if vpt != RG.launch_path(H)[0]:
            bad.append(("vpt", H, vpt))
            break
    body = " ".join(_one(r"static inline int row_threads\(int nvec\) \{(.*?)\n\}", read("common.cuh"), "row_threads").split())
    if body != ROW_THREADS:
        bad.append(("row_threads", body))
    return bad


def test_the_mirror_states_the_launchers():
    assert mismatches(CSRC) == []
    assert RG.STATIC_SMEM == {"rmsnorm": KG.STATIC_SMEM["rmsnorm_kernel"], "rmsnorm_quant": KG.STATIC_SMEM["rmsnorm_kernel<QUANT>"]}


@pytest.mark.parametrize("edit", [("elementwise.cu", "(nvec / 2) % 32 == 0 && nvec / 2 <= 256", "(nvec / 2) % 32 == 0 && nvec / 2 <= 128"),
                                  ("elementwise.cu", "nvec / 4 >= 64 && nvec / 4 <= 256", "nvec / 4 >= 32 && nvec / 4 <= 256"),
                                  ("elementwise.cu", "const int threads = row_threads(nvec);", "const int threads = row_threads(nvec / 2);"),
                                  ("elementwise.cu", "const size_t smem = (size_t)nvec * sizeof(uint4);",
                                   "const size_t smem = (size_t)nvec * 8;"),
                                  ("elementwise.cu", "    if (int e = fit_dynamic_smem<rmsnorm_kernel<T, FUSED, 0, QUANT>>(smem, what)) return e;\n", ""),
                                  ("elementwise.cu", "rmsnorm_kernel<T, FUSED, 4, QUANT><<<(unsigned)T_, nvec / 4,",
                                   "rmsnorm_kernel<T, FUSED, 4, QUANT><<<(unsigned)T_, nvec / 2,"),
                                  ("common.cuh", "nvec >= 256 ? 256", "nvec >= 128 ? 128")],
                         ids=["vpt2-range", "vpt4-range", "threads", "generic-smem", "generic-limit", "vpt4-threads", "row_threads"])
def test_a_changed_launcher_is_noticed(tmp_path, edit):
    f, old, new = edit
    for name in os.listdir(CSRC):
        if name.endswith((".cu", ".cuh")):
            shutil.copy(os.path.join(CSRC, name), tmp_path / name)
    text = (tmp_path / f).read_text()
    assert text.count(old) == 1
    (tmp_path / f).write_text(text.replace(old, new))
    assert mismatches(str(tmp_path)) != []


def test_the_width_table_covers_every_instance():
    by = {}
    for H in RG.WIDTHS:
        by.setdefault(RG.instance(H), []).append(H)
    assert sorted(by) == ["GEN", "GEN>48K", "VPT2", "VPT4"] and all(len(v) >= 2 for v in by.values()), by
    # both ends of each register instance's range, as the mirror computes them over every width the C ABI takes
    for vpt in (4, 2):
        Hs = [H for H in range(8, (1 << 16) + 1, 8) if RG.launch_path(H)[0] == vpt]
        assert min(Hs) in by[f"VPT{vpt}"] and max(Hs) in by[f"VPT{vpt}"], (vpt, min(Hs), max(Hs))
    assert (min(by["VPT2"]), max(by["VPT2"]), min(by["VPT4"]), max(by["VPT4"])) == (512, 3584, 2048, 8192)
    # the generic path: idle threads, several vectors per thread, the default 48 KB filled, exactly 48 KB of row and past it
    assert RG.launch_path(1040) == (0, 160, 130 * 16, False) and 1040 in by["GEN"]
    assert RG.launch_path(8200) == (0, 512, 1025 * 16, False) and 8200 in by["GEN"]
    assert RG.launch_path(24544) == (0, 512, 48 * 1024 - 64, False) and 24544 in by["GEN"]
    assert RG.launch_path(24552)[3] and RG.launch_path(24528, "rmsnorm_quant")[3]
    assert not RG.launch_path(24512, "rmsnorm_quant")[3]
    assert RG.launch_path(24576) == (0, 512, 48 * 1024, True) and 24576 in by["GEN>48K"]
    assert RG.launch_path(28672) == (0, 512, 3584 * 16, True) and 28672 in by["GEN>48K"]
    assert RG.launch_path(64) == (0, 32, 128, False)
    assert [RG.width_id(H) for H in (3584, 2048, 1040, 28672)] == ["VPT2-H3584", "VPT4-H2048", "GEN-H1040", "GEN>48K-H28672"]
    # the padded-divisor variant is only visible where the threads do not tile the row exactly
    assert [H for H in RG.WIDTHS if RG.padded_width(H) != H] == [64, 896, 1040, 8200, 24544, 24584]


def _rows(dt, H, fused):
    """The rows a GPU test normalises at width H (7 rows: every kind), and the weight."""
    x, r, w = RO.norm_inputs(7, H, dt, seed=H + 7 + 3 * fused, fused=fused)
    return (RO.add_residual(x, r) if fused else x), w


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("H", RG.WIDTHS, ids=RG.width_id)
def test_the_rmsnorm_bound_accepts_the_kernel_order_and_rejects_wrong_variants(H, dt, eps):
    vpt, threads, _, _ = RG.launch_path(H)
    for fused in (False, True):
        x, w = _rows(dt, H, fused)
        ok = lambda out: bool(RO.rmsnorm_ok(out, x, w, eps).all())
        assert ok(RO.rmsnorm_emulated(x, w, eps, vpt, threads)), "kernel order"
        assert ok(RO.rmsnorm_numpy_order(x, w, eps)), "numpy order"
        wrong = {"eps after sqrt": dict(eps_after_sqrt=True), "last warp dropped": dict(drop_last_warp=True),
                 "neighbour's rstd": dict(neighbour_rstd=True), "weight shifted a vector": dict(weight_shift=1)}
        if RG.padded_width(H) > 1.01 * H:      # at 24544 the padded mean is 0.13 % off: inside the fp32 sum's allowance
            wrong["mean over the padded width"] = dict(divisor=RG.padded_width(H))
        for name, kw in wrong.items():
            assert not ok(RO.rmsnorm_emulated(x, w, eps, vpt, threads, **kw)), name


def _all_finite(dt):
    v = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32).to(torch.int16).view(dt)
    return v[torch.isfinite(v.float())]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_the_silu_candidates_hold_the_fp32_formula_at_every_gate(dt):
    """Every finite 16-bit gate, up = 1 and up = 3: the reference kernel's fp32 formula meets the candidate check, and without
    the pinned band it fails exactly at the 17 bf16 gates -97, -96.5, ..., -89 (at no fp16 gate)."""
    gate = _all_finite(dt)[None, :]
    for u in (1.0, 3.0):
        x = torch.cat([torch.full_like(gate, u), gate], dim=1)
        out = RO.silu_and_mul_fp32(x)
        up = x[:, :gate.shape[1]]
        assert bool(RO.silu_and_mul_ok(out, up, gate).all())
        off = ~RO.silu_and_mul_ok(out, up, gate, pin_band=False)
        want = [] if dt == torch.float16 else [-97.0 + 0.5 * i for i in range(17)]
        assert sorted(gate[off].double().tolist()) == want


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_the_silu_data_rejects_a_single_rounding(dt):
    T, F = 33, 1032
    x = RO.silu_inputs(T, F, dt, seed=5)
    up, gate = x[:, :F], x[:, F:]
    g = gate.double()
    assert bool((g == -89).any() and (g == -97).any() and (g.abs() < 2.0 ** (-14 if dt == torch.float16 else -126)).any())
    assert bool((RO.bits(gate) == RO.bits(torch.tensor([-0.0], dtype=dt))).any()) and float(g.min()) >= -110 and float(g.max()) <= 20
    assert bool(RO.silu_and_mul_ok(RO.silu_and_mul_fp32(x), up, gate).all())
    assert not bool(RO.silu_and_mul_ok(RO.silu_and_mul_single_rounding(x), up, gate).all())


def test_round16_is_correct_rounding():
    for dt in DTYPES:
        v = _all_finite(dt).double()
        v = v[v.abs() < torch.finfo(dt).max]
        assert torch.equal(RO.bits(RO.round16(v, dt)), RO.bits(v.to(dt)))
        mid = (v[:-1] + v[1:]) / 2                      # ties between neighbours go to the even one
        assert torch.equal(RO.round16(mid, dt), mid.float().to(dt))
    assert float(RO.round16(torch.tensor([65520.0], dtype=torch.float64), torch.float16)) == np.inf
