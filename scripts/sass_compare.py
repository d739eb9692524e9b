"""Compare the machine code of two builds of a CUDA object, kernel by kernel (cuobjdump -sass; no GPU needed).

    python scripts/sass_compare.py OLD.o NEW.o [--rename 'NEW_NAME_REGEX=>REPLACEMENT' ...]

Kernels are matched by demangled name after the --rename substitutions are applied to the NEW build's names (for template
parameters a change added, e.g. the output type of the prepare kernels).  Instruction text is compared with addresses and
encodings stripped.  Prints one line per kernel of the OLD build (identical / DIFFERENT / missing) and exits 1 if any kernel of
the OLD build is missing or different in the NEW one."""
import argparse
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernels(obj):
    text = subprocess.run([CUOBJDUMP, "-sass", obj], check=True, capture_output=True, text=True).stdout
    out, name, body = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = body
            name, body = m.group(1), []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\*", line)
        if name and m:
            body.append(m.group(1))
    if name:
        out[name] = body
    mangled = list(out)
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.splitlines()
    return {d: out[m] for m, d in zip(mangled, demangled)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", action="append", default=[], help="REGEX=>REPLACEMENT applied to the new build's kernel names")
    a = ap.parse_args()
    old, new_raw = kernels(a.old), kernels(a.new)
    new = {}
    for name, body in new_raw.items():
        for r in a.rename:
            pat, rep = r.split("=>")
            name = re.sub(pat, rep, name)
        new.setdefault(name, body)
    bad = 0
    for name in sorted(old):
        if name not in new:
            print(f"missing    {name}")
            bad += 1
        elif new[name] != old[name]:
            print(f"DIFFERENT  {name}  ({len(old[name])} -> {len(new[name])} instructions)")
            bad += 1
        else:
            print(f"identical  {name}  ({len(old[name])} instructions)")
    print(f"{len(old) - bad} of {len(old)} kernels of {a.old} identical in {a.new}; {len(new_raw) - len(old)} more kernels in the new build")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
