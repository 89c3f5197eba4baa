"""The SASS and the resource usage of the objects build.py compiles, read with cuobjdump.  A test that reads an object
skips when cuobjdump or the object is absent."""
import functools
import os
import re
import shutil
import subprocess

import pytest

from internvideo_b200 import build


@functools.cache
def _dump(flag, obj):
    tool = next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)),
                None)
    if tool is None or not (build.OBJ / obj).exists():
        pytest.skip(f"needs cuobjdump and the built internvideo_b200/build/{obj}")
    return subprocess.run([tool, flag, str(build.OBJ / obj)], capture_output=True, text=True, check=True).stdout


def functions(obj):
    """{mangled kernel name: [SASS instruction lines]} of obj."""
    out, cur = {}, None
    for line in _dump("-sass", obj).splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line):
            out[cur].append(line)
    return out


def resources(obj):
    """{mangled kernel name: (registers, stack bytes, local bytes)} of obj."""
    return {m.group(1): tuple(map(int, m.group(2, 3, 4))) for m in
            re.finditer(r"Function (\S+):\s+REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _dump("-res-usage", obj))}


def count(lines, pattern):
    return sum(1 for l in lines if re.search(pattern, l))
