"""The recorded SASS of the library's kernels, tests/golden/kernel_sass.json: for each object build.py compiles, the
sha256 (first 16 hex digits) of every kernel's instructions as `cuobjdump -sass` prints them, with the address and
encoding comments stripped.  tests/test_dpe_abi_cpu.py holds every object the file lists to it, so a kernel whose
machine code changes by accident fails there.

After an intended change of a kernel's code (or a new nvcc), rebuild and rewrite the file from the new objects:

    python -m internvideo_b200.build && python tools/kernel_sass.py --write

A new object is not added unless it is named: python tools/kernel_sass.py --write --add ivb_new.o
"""
import argparse
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "kernel_sass.json"
sys.path.insert(0, str(ROOT))


def cuobjdump():
    return next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)),
                None)


def digest(lines):
    """The recorded form of one kernel's SASS instruction lines."""
    body = "\n".join(re.sub(r"/\*.*?\*/", "", l).strip() for l in lines)
    return hashlib.sha256(body.encode()).hexdigest()[:16]


def digests(path):
    """{mangled kernel name: digest} of one object file."""
    out = subprocess.run([cuobjdump(), "-sass", str(path)], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line):
            funcs[cur].append(line)
    return {k: digest(v) for k, v in funcs.items()}


def main():
    from internvideo_b200 import build
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="rewrite the golden file (else: compare and report)")
    ap.add_argument("--add", nargs="*", default=[], help="objects to record that the file does not list yet")
    a = ap.parse_args()
    golden = json.loads(GOLDEN.read_text())
    objs = sorted(set(golden) | set(a.add))
    now = {o: digests(build.OBJ / o) for o in objs}
    changed = {o: sorted(k for k in set(golden.get(o, {})) | set(now[o]) if golden.get(o, {}).get(k) != now[o].get(k))
               for o in objs}
    for o, ks in changed.items():
        if ks:
            print(f"{o}: {len(ks)} kernel(s) differ from the record")
    if a.write:
        GOLDEN.write_text(json.dumps(now, indent=1, sort_keys=True) + "\n")
        print(f"wrote {GOLDEN} ({sum(len(v) for v in now.values())} kernels in {len(now)} objects)")


if __name__ == "__main__":
    main()
