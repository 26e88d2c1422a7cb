"""Check that a refactor left the compiled kernels alone: pair the kernels of two builds by mangled name and compare
their SASS instruction by instruction, and their ptxas registers / stack / spills.

    nvcc -Xptxas=-v <the flags of unionml_b200/_build.py> -c X.cu -o OLD/X.o 2> OLD/X.ptxas.txt    # every .cu, both trees
    python tools/sass_diff.py OLD NEW [--skip REGEX] [--sub REGEX REPL]

--skip drops old kernels whose name matches (instantiations the change deletes); --sub rewrites the remaining old names
(e.g. a template argument the change removes) so that they pair with the new ones.  Instructions are compared without
their /*addr*/ and encoding comments.  A kernel that differs only in constant-bank offsets (a parameter struct that
lost fields) is reported as such.  Exit status 1 if anything else differs or a kernel has no partner.

    python tools/sass_diff.py --sizes DIR [--match REGEX]

prints, for every kernel of DIR/*.o (and of DIR/*.cubin), the bytes of SASS and the LDL / STL count of the kernel's own
code and of each out-of-line device function it calls (the ELF symbol table's ranges), so that code-size and
local-memory budgets can be checked without a GPU.  --match keeps the kernels whose name matches."""
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


def sass_by_addr(obj):  # kernel -> [(address, instruction)]
    out, name = {}, None
    text = subprocess.run(["cuobjdump", "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name and (m := re.match(r"\s*/\*([0-9a-f]{4,})\*/\s*(.*?)\s*;", line)):
            out[name].append((int(m.group(1), 16), m.group(2)))
    return out


def subfunctions(obj):  # kernel -> [(start, size, device function)]: the local FUNC symbols named $kernel$function
    out = {}
    text = subprocess.run(["cuobjdump", "-elf", str(obj)], capture_output=True, text=True, check=True).stdout
    for line in text.splitlines():
        m = re.match(r"\s*0x[0-9a-f]+\s+0x([0-9a-f]+)\s+0x([0-9a-f]+)\s+0x[0-9a-f]*2\s+\S+\s+\S+\s+\$(\S+?)\$(\S+)\s*$", line)
        if m:
            out.setdefault(m.group(3), []).append((int(m.group(1), 16), int(m.group(2), 16), m.group(4)))
    return out


def sizes(args):
    local = re.compile(r"\b(LDL|STL)(\.\S+)?\s")
    print(f"{'bytes':>8} {'LDL':>5} {'STL':>5}  function")
    for obj in sorted(args.old.glob("*.o")) + sorted(args.old.glob("*.cubin")):
        code, subs = sass_by_addr(obj), subfunctions(obj)
        for kernel in sorted(code):
            if args.match and not re.search(args.match, kernel):
                continue
            rest, lines = list(code[kernel]), []
            for start, size, fn in sorted(subs.get(kernel, [])):
                lines.append(([i for a, i in rest if start <= a < start + size], "    " + fn))
                rest = [(a, i) for a, i in rest if not start <= a < start + size]
            lines.insert(0, ([i for _, i in rest], f"{obj.stem}: {kernel} (own code; total {16 * len(code[kernel])})"))
            for body, label in lines:
                ldl = sum(1 for i in body if local.match(i + " ") and i.startswith("LDL"))
                stl = sum(1 for i in body if local.match(i + " ") and i.startswith("STL"))
                print(f"{16 * len(body):>8} {ldl:>5} {stl:>5}  {label}")
    return 0


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
    ap.add_argument("new", type=Path, nargs="?")
    ap.add_argument("--skip")
    ap.add_argument("--sub", nargs=2)
    ap.add_argument("--sizes", action="store_true")
    ap.add_argument("--match")
    args = ap.parse_args()
    if args.sizes:
        return sizes(args)
    if args.new is None:
        ap.error("two build directories are compared (or one with --sizes)")
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
