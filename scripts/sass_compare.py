#!/usr/bin/env python3
"""Per-kernel SASS comparison of two builds of the library (CPU only, needs cuobjdump on PATH or in /usr/local/cuda/bin): for every object file of `_build/fast` and `_build/strict`
under the first directory, the SASS of each function is compared with the same function in the second directory's object of the same name (instruction addresses dropped).  A change
that only adds kernels - a new pass whose arguments travel outside LaunchParams - leaves every function of the first build as it was.  Prints, per object, the functions that
changed and the ones that are new; exits 1 if any function of the first build changed or is missing.

    make -C <parent checkout>/rtxpt_b200/csrc _build/librtxpt_b200.so _build/librtxpt_b200_strict.so
    python scripts/sass_compare.py <parent checkout>/rtxpt_b200/csrc rtxpt_b200/csrc"""
import os
import re
import shutil
import subprocess
import sys


def cuobjdump():
    return shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def functions(obj):
    text = subprocess.run([cuobjdump(), "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m: cur = m.group(1); out[cur] = []; continue
        if cur: out[cur].append(re.sub(r"\s+", " ", re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)).strip())
    return out


def main():
    if len(sys.argv) != 3: sys.exit(__doc__)
    old_dir, new_dir = sys.argv[1:]
    bad = 0
    for variant in ("fast", "strict"):
        d = os.path.join(old_dir, "_build", variant)
        if not os.path.isdir(d): continue
        for name in sorted(f for f in os.listdir(d) if f.endswith(".o")):
            new_obj = os.path.join(new_dir, "_build", variant, name)
            if not os.path.exists(new_obj): print(f"{variant}/{name}: missing in {new_dir}"); bad += 1; continue
            a, b = functions(os.path.join(d, name)), functions(new_obj)
            changed = [f for f in a if a[f] != b.get(f)]
            added = [f for f in b if f not in a]
            print(f"{variant}/{name}: {len(a)} functions, {len(changed)} changed, {len(added)} new" + "".join(f"\n  changed: {f}" for f in changed) + "".join(f"\n  new: {f}" for f in added))
            bad += len(changed)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
