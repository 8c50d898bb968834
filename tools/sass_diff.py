"""Compare the SASS of two builds of libmaskflow_b200.so, function by function.

    python tools/sass_diff.py <so_a> <so_b>

Dumps both libraries with `cuobjdump -sass`, drops addresses, instruction encodings and comments, splits each dump per
function and diffs the instruction streams.  Prints a unified diff for every function that differs, the functions found on
one side only and a summary; exits 1 when anything differs.  For refactors that must leave the generated code alone (e.g.
moving device helpers between headers): build the parent and the change with the same Makefile and compare.  Two builds
of the same tree give identical dumps.
"""
import difflib
import os
import re
import shutil
import subprocess
import sys

COMMENT = re.compile(r"/\*.*?\*/")


def cuobjdump():
    return shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def functions(so):
    """{function name: [instruction lines]}; a name defined in several translation units gets a '#k' suffix."""
    out = subprocess.run([cuobjdump(), "-sass", so], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            key, k = name, 1
            while key in funcs:
                k += 1
                key = f"{name}#{k}"
            cur = funcs[key] = []
        elif line.startswith("Fatbin") or line.lstrip().startswith("code for"):
            cur = None
        elif cur is not None:
            text = " ".join(COMMENT.sub("", line).split())
            if text:
                cur.append(text)
    return funcs


def main(argv):
    if len(argv) != 3:
        sys.exit(__doc__)
    a, b = functions(argv[1]), functions(argv[2])
    differ = 0
    for name in sorted(a.keys() & b.keys()):
        if a[name] != b[name]:
            differ += 1
            sys.stdout.writelines(l + "\n" for l in difflib.unified_diff(a[name], b[name], name, name, n=1, lineterm=""))
    only = [("a", n) for n in sorted(a.keys() - b.keys())] + [("b", n) for n in sorted(b.keys() - a.keys())]
    for side, name in only:
        print(f"only in {side}: {name}")
    print(f"{len(a)} / {len(b)} functions, {differ} differ, {len(only)} on one side only")
    return 1 if differ or only else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
