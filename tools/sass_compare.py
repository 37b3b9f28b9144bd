"""Compares the kernels of two builds of the library: python tools/sass_compare.py old.so new.so

Prints one line per kernel: whether its SASS is identical, and REG / STACK / LOCAL of both builds.  Needs cuobjdump
(CUDA toolkit), no GPU.  Meant for refactors that should leave the generated code alone."""
from __future__ import annotations

import re
import shutil
import subprocess
import sys


def _cuobjdump(*args: str) -> str:
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return subprocess.run([exe, *args], check=True, capture_output=True, text=True).stdout


def sass(lib: str) -> dict[str, str]:
    """Kernel name -> its SASS text."""
    out: dict[str, list[str]] = {}
    cur = None
    for line in _cuobjdump("-sass", lib).splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
        elif cur is not None and "/*" in line:  # instructions and their encodings, not the section headers between kernels
            # cuobjdump pads every line to the widest instruction of the whole dump: compare the tokens, not the padding
            cur.append(" ".join(line.split()))
    return {k: "\n".join(v) for k, v in out.items()}


def res_usage(lib: str) -> dict[str, str]:
    """Kernel name -> "REG:n STACK:n LOCAL:n"."""
    text = _cuobjdump("-res-usage", lib)
    return {
        m.group(1): f"REG:{m.group(2)} STACK:{m.group(3)} LOCAL:{m.group(4)}"
        for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", text)
    }


def main(old: str, new: str) -> int:
    s_old, s_new = sass(old), sass(new)
    r_old, r_new = res_usage(old), res_usage(new)
    names = sorted(set(s_old) | set(s_new))
    n_diff = 0
    for name in names:
        if name not in s_old or name not in s_new:
            state = "only-old" if name in s_old else "only-new"
        else:
            state = "identical" if s_old[name] == s_new[name] else "different"
        n_diff += state != "identical"
        print(f"{state:9}  {r_old.get(name, '-'):24}  {r_new.get(name, '-'):24}  {name}")
    print(f"{len(names)} kernels, {n_diff} not identical")
    return 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__.splitlines()[0])
    sys.exit(main(sys.argv[1], sys.argv[2]))
