"""Check that a refactor left the compiled kernels alone: pair the kernels of two builds by mangled name and compare
their SASS instruction by instruction, and their ptxas registers / stack / spills.

    nvcc -Xptxas=-v <the flags of unionml_b200/_build.py> -c X.cu -o OLD/X.o 2> OLD/X.ptxas.txt    # every .cu, both trees
    python tools/sass_diff.py OLD NEW [--skip REGEX] [--sub REGEX REPL]

--skip drops old kernels whose name matches (instantiations the change deletes); --sub rewrites the remaining old names
(e.g. a template argument the change removes) so that they pair with the new ones.  Instructions are compared without
their /*addr*/ and encoding comments.  A kernel that differs only in constant-bank offsets (a parameter struct that
lost fields) is reported as such.  Exit status 1 if anything else differs or a kernel has no partner."""
import argparse
import re
import subprocess
import sys
from pathlib import Path

CBANK = re.compile(r"c\[0x0\]\[(0x[0-9a-f]+)\]")


def sass(obj):
    out, name = {}, None
    text = subprocess.run(["cuobjdump", "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name and (m := re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)):
            out[name].append(re.sub(r"\s+", " ", m.group(1)))
    return out


def resources(log):  # ptxas -v: entry function -> its stack / spill and register lines
    out, name = {}, None
    for line in Path(log).read_text().splitlines() if Path(log).exists() else []:
        if m := re.search(r"Compiling entry function '(\S+)'", line):
            name = m.group(1)
            out[name] = []
        elif name and re.search(r"Used \d+ registers|bytes stack frame", line):
            out[name].append(re.sub(r"^ptxas info\s*:", "", line).strip())
    return out


def paired(old, new, args):
    renamed = {}
    for name, v in old.items():
        if not (args.skip and re.search(args.skip, name)):
            renamed[re.sub(args.sub[0], args.sub[1], name) if args.sub else name] = v
    return renamed, new


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old", type=Path)
    ap.add_argument("new", type=Path)
    ap.add_argument("--skip")
    ap.add_argument("--sub", nargs=2)
    args = ap.parse_args()
    bad = same = offsets_only = 0
    for obj in sorted(args.old.glob("*.o")):
        old, new = paired(sass(obj), sass(args.new / obj.name), args)
        for name in sorted(set(old) | set(new)):
            if name not in old or name not in new:
                print(f"{obj.stem}: only in {'new' if name in new else 'old'}: {name}")
                bad += 1
            elif old[name] == new[name]:
                same += 1
            else:
                diffs = [(x, y) for x, y in zip(old[name], new[name]) if x != y]
                if len(old[name]) == len(new[name]) and all(CBANK.sub("c[]", x) == CBANK.sub("c[]", y) for x, y in diffs):
                    moved = sorted({(CBANK.findall(x)[0], CBANK.findall(y)[0]) for x, y in diffs})
                    print(f"{obj.stem}: {name}: constant-bank offsets only {moved}")
                    offsets_only += 1
                else:
                    print(f"{obj.stem}: {name}: {len(diffs)} of {len(old[name])} instructions differ")
                    bad += 1
        old, new = paired(resources(obj.with_suffix(".ptxas.txt")), resources(args.new / (obj.stem + ".ptxas.txt")), args)
        for name in sorted(set(old) & set(new)):
            if old[name] != new[name]:
                print(f"{obj.stem}: {name}: ptxas {old[name]} -> {new[name]}")
                bad += 1
    print(f"{same} kernels identical, {offsets_only} differ in constant-bank offsets only, {bad} other differences")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
