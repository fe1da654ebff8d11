"""Compare the SASS of kernels in two builds of the same source, e.g. before and after a refactor that should not change the
machine code.  Each OLD=NEW argument is a pair of regular expressions that each match one mangled kernel name.
  python tools/sass_diff.py before.o after.o 'blend_fwd_kernelILb0ELb0E=blend_fwd_kernelILb0E' ...
Prints, per pair, whether the opcode sequences are identical and every instruction whose operands differ (addresses and
encodings stripped).  Exits 1 when an opcode sequence differs."""
import re
import subprocess
import sys


def kernels(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = fns.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s*(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return fns


def find(fns, pattern):
    hits = [k for k in fns if re.search(pattern, k)]
    if len(hits) != 1:
        sys.exit(f"{pattern!r} matches {len(hits)} kernels: {hits}")
    return fns[hits[0]]


def opcodes(sass):
    return [re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0] for ins in sass]


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    same = True
    for pair in sys.argv[3:]:
        a, b = (find(fns, p) for fns, p in zip((old, new), pair.split("=")))
        diff = [(x, y) for x, y in zip(a, b) if x != y]
        ok = opcodes(a) == opcodes(b)
        same &= ok
        print(f"{pair}: {len(a)} -> {len(b)} instructions, opcodes {'identical' if ok else 'DIFFER'}, "
              f"{len(diff)} with other operands")
        for x, y in diff:
            print(f"  - {x}\n  + {y}")
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
