"""Per-kernel SASS comparison of two builds of libehb200.so.

    python tools/sass_diff.py OLD.so NEW.so

Disassembles both libraries with cuobjdump -sass, splits the listing per function, and prints the kernels that
exist in only one of them and those whose instructions differ (addresses and encodings stripped; the translation
unit hash in anonymous-namespace names is ignored).  Exit status 1
when a kernel of OLD is missing from NEW or differs.
"""
import re
import subprocess
import sys


def kernels(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            # anonymous-namespace names carry a hash of the translation unit, which changes with any header it reads
            name = re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+_\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1", m.group(1))
            funcs[name] = []
            continue
        if name is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m:
            funcs[name].append(m.group(1).strip())
    return funcs


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    missing = sorted(set(old) - set(new))
    added = sorted(set(new) - set(old))
    changed = sorted(n for n in set(old) & set(new) if old[n] != new[n])
    for n in missing:
        print("missing:", n)
    for n in changed:
        print("changed:", n)
    for n in added:
        print("added:  ", n)
    print(f"{len(old)} kernels before, {len(new)} after: {len(changed)} changed, {len(missing)} missing, "
          f"{len(added)} added")
    return 1 if missing or changed else 0


if __name__ == "__main__":
    sys.exit(main())
