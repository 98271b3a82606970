"""Compare two builds of libiggt_b200.so kernel by kernel (no GPU needed): the SASS instruction text of every kernel,
without instruction offsets and encodings, and its `cuobjdump -res-usage` line (registers, shared memory, stack).
Prints the kernels that exist in one build only and the kernels that differ; exits 1 if there are any.

    python scripts/sass_diff.py parent/libiggt_b200.so branch/libiggt_b200.so
"""
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
INSN = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;")


def _run(flag, lib):
    return subprocess.run([CUOBJDUMP, flag, lib], check=True, capture_output=True, text=True).stdout.splitlines()


def kernels(lib):
    """{kernel name: (instruction list, resource-usage line)}"""
    sass, name = {}, None
    for line in _run("-sass", lib):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            if name in sass:
                raise SystemExit(f"{lib}: kernel {name} appears twice")
            sass[name] = []
            continue
        m = INSN.match(line)
        if m and name:
            sass[name].append(" ".join(m.group(1).split()))
    res, name = {}, None
    for line in _run("-res-usage", lib):
        m = re.match(r"\s*Function (\S+):$", line)
        if m:
            name = m.group(1)
        elif name and line.strip().startswith("REG:"):
            res[name] = line.strip()
            name = None
    return {k: (v, res.get(k)) for k, v in sass.items()}


def main(argv):
    if len(argv) != 3:
        raise SystemExit(__doc__)
    a, b = kernels(argv[1]), kernels(argv[2])
    only_a, only_b = sorted(a.keys() - b.keys()), sorted(b.keys() - a.keys())
    common = sorted(a.keys() & b.keys())
    print(f"{len(a)} kernels in {argv[1]}, {len(b)} in {argv[2]}, {len(common)} in both")
    for name in only_a:
        print(f"only in {argv[1]}: {name}")
    for name in only_b:
        print(f"only in {argv[2]}: {name}")
    differ = 0
    for name in common:
        (sa, ra), (sb, rb) = a[name], b[name]
        what = [w for w, same in (("sass", sa == sb), ("resources", ra == rb)) if not same]
        if what:
            differ += 1
            detail = f" ({len(sa)} vs {len(sb)} instructions)" if "sass" in what else ""
            print(f"differs ({', '.join(what)}){detail}: {name}")
            if "resources" in what:
                print(f"    {ra}\n    {rb}")
    print(f"{differ} kernels differ")
    return 1 if only_a or only_b or differ else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
