"""Compare the SASS of two builds function by function.

    python scripts/sass_diff.py OLD.so|.o NEW.so|.o

Runs `cuobjdump -sass` on both files and compares each function's instruction and encoding lines, ignoring whitespace (the
headers and section banners are not compared).  Prints the counts of identical, differing, removed and added functions and
names every function that is not identical.  Exits 1 when a function differs or disappears, 0 otherwise: a refactor that
claims to move no instruction must leave every function identical.

CUOBJDUMP overrides the cuobjdump binary (default: the one on PATH, else /usr/local/cuda/bin/cuobjdump).
"""
import os
import re
import shutil
import subprocess
import sys

FUNCTION = re.compile(r"^\s*Function\s*:\s*(\S+)")
# "/*0040*/  UIADD3 UR4, UR4, 0xff, URZ ;  /* 0x000000ff04047890 */" and the encoding's second half "/* 0x000fe2000fffe03f */"
CODE = re.compile(r"^\s*/\*(?:[0-9a-f]{4,}\*/|\s*0x[0-9a-f]{16}\s*\*/)")


def cuobjdump():
    return os.environ.get("CUOBJDUMP") or shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def functions(path):
    """{function name: [code lines without whitespace]}; a name met again (another cubin) gets a '#n' suffix."""
    r = subprocess.run([cuobjdump(), "-sass", path], capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(f"cuobjdump -sass {path} failed:\n{r.stderr}")
    out, cur = {}, None
    for line in r.stdout.splitlines():
        m = FUNCTION.match(line)
        if m:
            name, n = m.group(1), 1
            while (name if n == 1 else f"{name}#{n}") in out:
                n += 1
            cur = out.setdefault(name if n == 1 else f"{name}#{n}", [])
        elif cur is not None and CODE.match(line):
            cur.append("".join(line.split()))
    return out


def main(argv):
    if len(argv) != 3:
        sys.exit(__doc__)
    old, new = functions(argv[1]), functions(argv[2])
    same = sorted(f for f in old if f in new and old[f] == new[f])
    differ = sorted(f for f in old if f in new and old[f] != new[f])
    removed = sorted(f for f in old if f not in new)
    added = sorted(f for f in new if f not in old)
    print(f"{len(same)} identical, {len(differ)} differing, {len(removed)} removed, {len(added)} added "
          f"({len(old)} functions before, {len(new)} after)")
    for tag, names in (("differs", differ), ("removed", removed), ("added", added)):
        for f in names:
            print(f"  {tag}: {f}")
    return 1 if differ or removed else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
