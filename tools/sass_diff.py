#!/usr/bin/env python3
"""Compare two builds of a CUDA module function by function, by mangled name:

    python tools/sass_diff.py OLD.so NEW.so [--list]

Every function present in both must have the same instructions (`cuobjdump -sass`) and the same resource usage
(`cuobjdump -res-usage`).  Prints the number of common, changed, removed and added functions (--list: the removed and the added
ones, demangled).  Exit status 1 when a common function changed or a function was added."""
import collections
import re
import subprocess
import sys

INSN = re.compile(r"^\s+/\*(?:[0-9a-f]{4,}\*/|\s*0x[0-9a-f]+\s*\*/)")


def functions(path):
    """mangled name -> sorted list of (instructions, resource usage), one entry per cubin that contains the function"""
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", path], capture_output=True, text=True, check=True).stdout
    usage = collections.defaultdict(list)
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            usage[cur].append(line.strip())
            cur = None
    code = collections.defaultdict(list)
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        # whitespace normalised: cuobjdump pads the encoding column to the longest instruction of the cubin
        code[name.strip()].append("\n".join(" ".join(ln.split()) for ln in body.splitlines() if INSN.match(ln)))
    return {n: sorted(zip(c, sorted(usage[n]) or [""] * len(c))) for n, c in code.items()}


def demangle(names):
    return subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines() if names else []


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    if len(args) != 2:
        sys.exit(__doc__)
    old, new = functions(args[0]), functions(args[1])
    common = sorted(old.keys() & new.keys())
    changed = [n for n in common if old[n] != new[n]]
    removed, added = sorted(old.keys() - new.keys()), sorted(new.keys() - old.keys())
    print(f"common {len(common)}  changed {len(changed)}  removed {len(removed)}  added {len(added)}")
    for title, names in (("changed", changed), ("added", added)) + ((("removed", removed),) if "--list" in sys.argv else ()):
        for n in demangle(names):
            print(f"{title}: {n}")
    sys.exit(1 if changed or added else 0)


if __name__ == "__main__":
    main()
