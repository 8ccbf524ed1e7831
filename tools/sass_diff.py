#!/usr/bin/env python3
"""Compare the SASS of two builds symbol by symbol (CPU only).

    python tools/sass_diff.py a.cubin b.cubin        (or two .so files)

Disassembles both with `cuobjdump -sass`, splits the listing at every `Function :` header and compares each kernel's
instructions.  Prints the symbol counts, how many are identical and the demangled names of those that differ, are
missing from b or are new in b.  Exits 1 on any such symbol, so identical SASS (hence identical registers, spills and
schedule) can be required of a change that should not alter the generated code.
"""
import os
import re
import shutil
import subprocess
import sys


def tool(name):
    found = shutil.which(name)
    return found or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)


def functions(path):
    out = subprocess.run([tool("cuobjdump"), "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
        elif cur is not None and line.strip():
            cur.append(" ".join(line.split()))      # cuobjdump pads columns to the widest line of the whole file
    return funcs


def demangle(names):
    if not names:
        return []
    return subprocess.run([tool("cu++filt")], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")[: len(names)]


def main(argv):
    if len(argv) != 3:
        sys.exit(__doc__)
    a, b = functions(argv[1]), functions(argv[2])
    common = [k for k in a if k in b]
    differ = [k for k in common if a[k] != b[k]]
    missing, new = [k for k in a if k not in b], [k for k in b if k not in a]
    print(f"symbols: {len(a)} vs {len(b)}; identical {len(common) - len(differ)}, differing {len(differ)}, "
          f"missing {len(missing)}, new {len(new)}")
    for tag, names in (("differs", differ), ("missing", missing), ("new", new)):
        for k, name in zip(names, demangle(names)):
            extra = f" ({len(a[k])} vs {len(b[k])} lines)" if tag == "differs" else ""
            print(f"  {tag}: {name}{extra}")
    return 1 if differ or missing or new else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
