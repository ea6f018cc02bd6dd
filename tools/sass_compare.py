#!/usr/bin/env python
"""Compares the SASS of two builds of the library function by function (no GPU needed).

    python tools/sass_compare.py OLD.so NEW.so

cuobjdump -sass of both files, split into functions, names demangled.  A function of OLD must exist in NEW with the
same instructions and encodings.  The any-hit and multi-hit template parameters of the warp-queue kernel (kAnyHit and
kMultiHit, default false) only change the symbol names of the instantiations that leave them false; they are mapped out
of the names of both builds before the comparison, so OLD may be a build from before or after the any-hit or multi-hit
variants (it needs ray mode, kRays).  Functions that exist in NEW only are listed.  Exit code 0 = every function of OLD
is identical.
"""
import collections
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def functions(path):
    text = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    out, name, body = collections.OrderedDict(), None, []
    seen = collections.Counter()

    def close():
        if name is not None:
            seen[name] += 1
            out[(name, seen[name])] = body

    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            close()
            name, body = m.group(1), []
        elif name is not None and line.strip() and not line.strip().startswith("."):
            body.append(line.strip())
    close()
    names = sorted({k[0] for k in out})
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    d = dict(zip(names, dem))
    return collections.OrderedDict(((d[n], i), b) for (n, i), b in out.items())


def normalise(name):
    # render_warpqueue_kernel<K, kSpread, kPacket, kAllNodes, kSpheres, kRays, kAnyHit, false>(...)
    # -> the name the same instantiation had before the multi-hit parameter existed, then
    # render_warpqueue_kernel<K, kSpread, kPacket, kAllNodes, kSpheres, kRays, false>(...)
    # -> the name it had before the any-hit parameter existed
    for n_before in (7, 6):
        name = re.sub(r"render_warpqueue_kernel<((?:[^,<>]+, ){%d}[^,<>]+), false>\(" % (n_before - 1),
                      r"render_warpqueue_kernel<\1>(", name)
    return name


def main():
    old, new = ({(normalise(n), i): b for (n, i), b in functions(path).items()} for path in sys.argv[1:3])
    bad = 0
    for key, body in old.items():
        other = new.get(key)
        if other is None:
            print(f"MISSING  {key[0]}")
            bad += 1
        elif other != body:
            diff = sum(a != b for a, b in zip(body, other)) + abs(len(body) - len(other))
            print(f"DIFFERS  {key[0]}  ({len(body)} -> {len(other)} lines, {diff} differ)")
            bad += 1
    added = [n for (n, _) in new if (n, 1) not in old]
    print(f"{len(old)} functions compared, {bad} not identical; {len(added)} new:")
    for n in added:
        print(f"NEW      {n}")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
