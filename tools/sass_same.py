"""Check that two builds of libspconv.so hold the same device code:

    python tools/sass_same.py OLD.so NEW.so

Splits each `cuobjdump -sass` listing at its `Function :` headers and compares the sets of (kernel name, instruction
text).  The ids nvcc puts in the names of anonymous namespaces depend on where a file was compiled, so they are
dropped (_GLOBAL__N__<id>_14_conv_direct_cu_<id> becomes _GLOBAL__N__14_conv_direct_cu).  A function's text is its
instruction and label lines; the listing's per-file headers (source paths, fatbin sections) are not part of it.  A
host-only change must leave the sets identical: same kernels, same SASS.  Exit status 0 when they are.
"""
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def kernels(path):
    out = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    out = re.sub(r"\d*_GLOBAL__N__[0-9a-f]{8}_(\d+_\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1", out)
    funcs = {}
    for part in re.split(r"^\s*Function : ", out, flags=re.M)[1:]:
        name, _, body = part.partition("\n")
        funcs[name.strip()] = "\n".join(ln.strip() for ln in body.splitlines() if ln.strip().startswith(("/*", ".L")))
    return funcs


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    gone, added = sorted(old.keys() - new.keys()), sorted(new.keys() - old.keys())
    changed = sorted(k for k in old.keys() & new.keys() if old[k] != new[k])
    for tag, names in (("only in old", gone), ("only in new", added), ("different SASS", changed)):
        for n in names:
            print("%s: %s" % (tag, n))
    print("%d kernels in old, %d in new; %d differ" % (len(old), len(new), len(gone) + len(added) + len(changed)))
    sys.exit(1 if gone or added or changed else 0)


if __name__ == "__main__":
    main()
