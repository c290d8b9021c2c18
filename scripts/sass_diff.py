#!/usr/bin/env python
"""Compare the SASS of every kernel in swiftllm_b200/csrc/build/*.o with a saved baseline.

    python scripts/sass_diff.py save  <dir>      # dump one normalised .sass per kernel into <dir>
    python scripts/sass_diff.py check <dir>      # report kernels whose instruction stream changed / appeared / vanished
    python scripts/sass_diff.py manifest <json> "<where validated>"   # hash of every kernel's normalised SASS: written after the
                                                 # whole `pytest -m gpu` suite, smoke() and bench.py passed on an H100 with this
                                                 # exact build (tests/test_cabi.py holds later builds to it)

Used when a validated kernel's SOURCE is refactored without a GPU at hand (e.g. moved into a shared template): an
unchanged instruction stream means the GPU validation of that kernel still stands.  Mangled names are normalised by
dropping template arguments that were added, so compare by demangled prefix when a template parameter was appended.
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "swiftllm_b200", "csrc", "build")


def kernels():
    out = {}
    for f in sorted(os.listdir(OBJ)):
        if not f.endswith(".o"):
            continue
        txt = subprocess.run(["cuobjdump", "-sass", os.path.join(OBJ, f)], capture_output=True, text=True).stdout
        name, body = None, []
        for line in txt.splitlines():
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                if name:
                    out[name] = body
                name, body = m.group(1), []
                continue
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
            if m and name:
                body.append(m.group(1).strip())
        if name:
            out[name] = body
    return out


def norm(body):
    """Instruction stream with the offsets into constant bank 4 (module-level constants: printf format strings, globals)
    blanked: adding an unrelated kernel with its own strings to a translation unit shifts them."""
    return [re.sub(r"c\[0x4\]\[0x[0-9a-f]+\]", "c[0x4][*]", i) for i in body]


def demangle(names):
    r = subprocess.run(["cu++filt"] + list(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, r))


def main():
    mode, d = sys.argv[1], sys.argv[2]
    ks = kernels()
    if mode == "manifest":
        import hashlib
        import json
        dm = demangle(sorted(ks))
        nvcc = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
        rel = re.search(r"release [0-9.]+, V[0-9.]+", nvcc)
        man = {"nvcc": rel.group(0) if rel else nvcc.strip().splitlines()[-1], "flags": "see swiftllm_b200/build.py",
               "validated_at": sys.argv[3] if len(sys.argv) > 3 else "",
               "kernels": {dm[n]: {"sha256": hashlib.sha256("\n".join(norm(b)).encode()).hexdigest(), "instructions": len(b)}
                           for n, b in sorted(ks.items())},
               "equivalent": {}}
        json.dump(man, open(d, "w"), indent=1)
        print(f"manifest of {len(ks)} kernels -> {d}")
        return
    if mode == "save":
        os.makedirs(d, exist_ok=True)
        for n, b in ks.items():
            open(os.path.join(d, n + ".sass"), "w").write("\n".join(b) + "\n")
        print(f"saved {len(ks)} kernels")
        return
    base = {f[:-5]: open(os.path.join(d, f)).read().splitlines() for f in os.listdir(d) if f.endswith(".sass")}
    dm = demangle(sorted(set(ks) | set(base)))
    same = changed = 0
    for n in sorted(base):
        if n in ks:
            if ks[n] == base[n]:
                same += 1
            elif norm(ks[n]) == norm(base[n]):
                same += 1
                print(f"same*    {dm[n]}  (identical up to constant-bank-4 offsets, i.e. addresses of printf strings / globals)")
            else:
                changed += 1
                d = sum(1 for x, y in zip(ks[n], base[n]) if x != y) + abs(len(ks[n]) - len(base[n]))
                print(f"CHANGED  {dm[n]}  ({len(base[n])} -> {len(ks[n])} instructions, {d} differ)")
        else:
            # a template parameter may have been appended: match on identical instruction streams
            twins = [m for m in ks if m not in base and norm(ks[m]) == norm(base[n])]
            if twins:
                same += 1
                print(f"renamed  {dm[n]}  ->  {dm[twins[0]]}  (identical instructions)")
            else:
                changed += 1
                print(f"MISSING  {dm[n]}")
    new = [n for n in ks if n not in base]
    print(f"{same} identical, {changed} changed/missing, {len(new)} new kernels")
    for n in new:
        print(f"new      {dm[n]}")


if __name__ == "__main__":
    main()
