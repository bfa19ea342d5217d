"""(CPU) Compare the machine code of two builds of the library, kernel by kernel.

    python tools/sass_compare.py OLD.so NEW.so

Runs ``cuobjdump -sass`` on both libraries, splits each listing at its ``Function :`` headers and reports every
kernel as identical, different or missing (present in one library only).  Runs of blanks are compared as one: the
listing pads its columns to the widest instruction of the whole library, so a new kernel can re-pad unchanged ones.
Exits 1 unless every kernel is identical.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys


def kernels(so: str) -> dict[str, str]:
    """Kernel name -> its SASS text, from ``cuobjdump -sass so``."""
    cuobjdump = os.environ.get("CUOBJDUMP", "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", so], check=True, capture_output=True, text=True).stdout
    out = {}
    parts = re.split(r"^\s*Function : (\S+)\s*$", text, flags=re.M)
    for name, body in zip(parts[1::2], parts[2::2]):
        out[name] = re.sub(r"[ \t]+", " ", body)
    return out


def main(argv: list[str]) -> int:
    if len(argv) != 3:
        print(__doc__.strip(), file=sys.stderr)
        return 2
    old, new = kernels(argv[1]), kernels(argv[2])
    bad = 0
    for name in sorted(old.keys() | new.keys()):
        if name not in old or name not in new:
            verdict = f"missing from {'OLD' if name not in old else 'NEW'}"
        else:
            verdict = "identical" if old[name] == new[name] else "different"
        bad += verdict != "identical"
        print(f"{verdict:18} {name}")
    print(f"{len(old.keys() | new.keys())} kernels, {bad} not identical")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
