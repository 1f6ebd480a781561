#!/usr/bin/env python
"""Per-kernel SASS of two builds of the library, compared: which kernels are byte-identical, changed, missing or new.

  python tools/sass_diff.py OLD.so NEW.so

Each library is disassembled with `cuobjdump -sass`; the source-file identifier lines are dropped and runs of blanks
collapsed, so two builds of the same code in different directories, or next to different kernels, compare equal.  Exit status 1 when a kernel of OLD is changed or missing."""
import re
import subprocess
import sys


def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and not line.startswith("identifier =") and "Fatbin" not in line \
                and "code for sm_" not in line:
            # runs of blanks collapsed: cuobjdump pads its columns to the widest instruction of the whole
            # module, so a new kernel in the same file would otherwise shift an unchanged kernel's lines
            funcs[cur].append(" ".join(line.split()))
    return {k: "\n".join(v) for k, v in funcs.items()}


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    changed = [k for k in old if k in new and old[k] != new[k]]
    missing = [k for k in old if k not in new]
    added = [k for k in new if k not in old]
    print(f"{len(old)} kernels in {sys.argv[1]}: {len(old) - len(changed) - len(missing)} identical, "
          f"{len(changed)} changed, {len(missing)} missing; {len(added)} new")
    for tag, names in (("changed", changed), ("missing", missing), ("new", added)):
        for k in names:
            print(f"  {tag}: {k}")
    return 1 if changed or missing else 0


if __name__ == "__main__":
    sys.exit(main())
