"""Compare the machine code of two builds of libkiss_icp_b200.so kernel by kernel.

    python tools/sass_diff.py OLD.so NEW.so

Every kernel of both libraries (cuobjdump -sass) is matched by its source file and demangled name. A parameter type
that moved to kb_types (csrc/types.cuh) is read as the module's own type, so that k_fs_index(kb_fs::MapView, ...) and
k_fs_index(kb_types::MapView, ...) are the same kernel. Prints one line per kernel that is missing on either side or
whose instruction stream differs, then a summary; exits 1 when anything differs. Instructions are compared with their
encodings, without the addresses cuobjdump prints in front of them.
"""
from __future__ import annotations

import re
import subprocess
import sys


def kernels(lib: str) -> dict[str, list[str]]:
    sass = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    out: dict[str, list[str]] = {}
    name = unit = None
    for line in sass.splitlines():
        u = re.match(r"identifier = .*?(\w+\.cu)$", line)
        if u:
            unit = u.group(1)
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = f"{unit} {m.group(1)}"
            if name in out:
                raise SystemExit(f"{lib}: {name} appears twice")
            out[name] = []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            out[name].append(re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", line).strip())
        elif name and re.match(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", line):  # second half of an instruction's encoding
            out[name].append(line.strip())
    return out


def keyed(lib: str) -> dict[str, list[str]]:
    ks = kernels(lib)
    names = subprocess.run(["c++filt"], input="\n".join(ks), check=True, capture_output=True, text=True).stdout.split("\n")
    out = {}
    for mangled, demangled in zip(ks, names):
        ns = re.match(r"\S+ (?:void )?(kb\w*)::", demangled)
        key = demangled.replace("kb_types::", ns.group(1) + "::") if ns else demangled
        if key in out:
            raise SystemExit(f"{lib}: {key} appears twice")
        out[key] = ks[mangled]
    return out


def main() -> int:
    old, new = keyed(sys.argv[1]), keyed(sys.argv[2])
    bad = 0
    for k in sorted(set(old) | set(new)):
        if k not in new:
            print("only in old:", k)
        elif k not in old:
            print("only in new:", k)
        elif old[k] != new[k]:
            print(f"differs ({len(old[k])} vs {len(new[k])} lines):", k)
        else:
            continue
        bad += 1
    print(f"{len(old)} kernels in old, {len(new)} in new, {bad} missing or different")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
