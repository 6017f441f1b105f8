"""Compare two `cuobjdump -sass` listings function by function, addresses and encodings ignored.

    python scripts/compare_sass.py OLD.sass NEW.sass

Each `Function :` section's instructions are compared under the function's mangled name, with the per-build hash of
anonymous namespaces (`_GLOBAL__N__<8 hex digits>_`) normalised, the `/*0123*/` addresses and the `/* 0x... */` encodings
stripped.  Prints the counts of identical, changed, removed and added functions, then every changed, removed and added
name (demangled when c++filt is on the PATH).  Exit code 0.
"""
from __future__ import annotations

import re
import shutil
import subprocess
import sys


def functions(path):
    out, cur = {}, None
    for line in open(path):
        m = re.match(r"\s*Function : (\S+)", re.sub(r"_GLOBAL__N__[0-9a-f]{8}_", "_GLOBAL__N__X_", line))
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        if cur is None:
            continue
        body = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)).strip()
        if body:
            out[cur].append(body)
    return out


def demangle(name):
    if not shutil.which("c++filt"):
        return name
    return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    same = [n for n in old if n in new and old[n] == new[n]]
    changed = [n for n in old if n in new and old[n] != new[n]]
    removed = [n for n in old if n not in new]
    added = [n for n in new if n not in old]
    print(f"old {len(old)}, new {len(new)}: identical {len(same)}, changed {len(changed)}, removed {len(removed)}, "
          f"added {len(added)}")
    for tag, names in (("CHANGED", changed), ("REMOVED", removed), ("ADDED", added)):
        for n in names:
            print(tag, demangle(n))


if __name__ == "__main__":
    main()
