"""Compares the kernels of two builds of libbvh_b200.so instruction by instruction.

    python tools/sass_diff.py OLD.so NEW.so

Splits `cuobjdump -sass` into one body per function, drops the instruction addresses and encodings (SASS branch targets are already
relative to the function) and masks the 32@lo / 32@hi relocations of symbol addresses.  A name can occur in more than one translation
unit, so each build is a multiset of (name, body) pairs.  Reports, per name, the bodies only one build has.  Exit code 0 when both
builds hold the same multiset.  A host-only change (drivers, entry points) must leave every kernel identical."""
import collections
import re
import subprocess
import sys

_FUNC = re.compile(r"^\s*Function : (\S+)\s*$")
_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s*(.*?)\s*;?\s*(?:/\*.*\*/)?\s*$")


def bodies(path):
    """Counter of (name, normalised body) over every function of the file."""
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, name, body = collections.Counter(), None, []
    for line in out.splitlines():
        m = _FUNC.match(line)
        if m:
            if name:
                funcs[(name, normalise(body))] += 1
            name, body = m.group(1), []
            continue
        m = _INSN.match(line)
        if name and m:
            body.append(m.group(2))
    if name:
        funcs[(name, normalise(body))] += 1
    return funcs


def normalise(body):
    return tuple(re.sub(r"\b(32@lo|32@hi)\([^)]*\)", r"\1(sym)", i) for i in body)


def main(old, new):
    a, b = bodies(old), bodies(new)
    only_a, only_b = a - b, b - a
    print(f"functions: {sum(a.values())} in {old} ({len({k[0] for k in a})} names), {sum(b.values())} in {new} "
          f"({len({k[0] for k in b})} names); bodies only in old {sum(only_a.values())}, only in new {sum(only_b.values())}")
    for k in sorted({k[0] for k in only_a} | {k[0] for k in only_b}):
        print("  differs:", k)
    return 1 if only_a or only_b else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
