#!/usr/bin/env python
"""Compares the SASS of two builds of one source file kernel by kernel: every kernel of OLD must have the same
instructions, in the same order, as the same-named kernel of NEW (the encoding comments are ignored); kernels only NEW
has are counted. Exit status 1 on any difference or any kernel NEW lacks. Runs on the build box (cuobjdump, no GPU).

    nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O3 -lineinfo -Xcompiler -fPIC -I include \\
         -I bevformer_tensorrt_b200/csrc -c bevformer_tensorrt_b200/csrc/bev_pool.cu -o new.o   # and old.o at the parent
    python scripts/sass_diff.py old.o new.o
"""
import re
import subprocess
import sys


# the tag of an anonymous namespace, which encodes the source file's name and a hash: <len>_GLOBAL__N__<hash>_<file>_<hash>
_ANON = re.compile(r"\d+_GLOBAL__N__\w+?_[0-9a-f]{8}(?=\d)")


def kernels(obj):
    """{mangled kernel name, its anonymous-namespace tag dropped: [instruction text, ...]} of an object file or shared
    library."""
    text = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = _ANON.sub("_GLOBAL__N_", m.group(1))
            out[name] = []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            out[name].append(re.sub(r"\s*/\* 0x[0-9a-f]+ \*/", "", line).strip())
    return out


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    differ = [k for k, body in old.items() if new.get(k) != body]
    for k in differ:
        print("differs:" if k in new else "missing:", k)
    print(f"{len(old)} kernels in {sys.argv[1]}: {len(old) - len(differ)} identical; {len(set(new) - set(old))} new")
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
