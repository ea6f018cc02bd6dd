#!/usr/bin/env python
"""Compares the SASS of two builds of the library function by function (no GPU needed).

    python tools/sass_compare.py OLD.so NEW.so

cuobjdump -sass of both files, split into functions, names demangled.  A function of OLD must exist in NEW with the
same instructions and encodings.  The warp-queue kernel's instantiations are matched by one canonical key, (K, spread,
packet, all-nodes, spheres, query kind, ranged, accum, views), parsed from every form its template has had: five
parameters (pixel frames only), six (kRays), seven (kAnyHit), eight (kMultiHit), the query-kind enum (Query), the enum
followed by kRanged (per-ray intervals), by kRanged and kAccum (progressive rendering) and by kRanged, kAccum and kViews
(several views in one launch); a parameter a form does not have is false.  So OLD and NEW may be builds of any of them.  Functions that exist in NEW only are listed.  Exit code 0 = every function of OLD is identical.
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
            body.append(" ".join(line.split()))   # cuobjdump pads its columns to the widest line of the whole file
    close()
    names = sorted({k[0] for k in out})
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    d = dict(zip(names, dem))
    return collections.OrderedDict(((d[n], i), b) for (n, i), b in out.items())


WARPQUEUE = re.compile(r"render_warpqueue_kernel<([^<>]*)>\(")
KINDS = ("pixels", "closest", "any-hit", "multi-hit")   # the values of the Query enum, in order


def canonical(name):
    """The key of a warp-queue instantiation, whatever the form of its template; other names as they are."""
    m = WARPQUEUE.search(name)
    if not m:
        return name
    args = [a.strip() for a in m.group(1).split(",")]
    k, (spread, packet, all_nodes, spheres), rest = args[0], args[1:5], args[5:]
    enum = re.fullmatch(r"\(.*Query\)(\d+)", rest[0]) if rest else None
    ranged = accum = views = False
    if enum:   # <K, kSpread, kPacket, kAllNodes, kSpheres, (Query)N[, kRanged[, kAccum[, kViews]]]>
        kind = KINDS[int(enum.group(1))]
        ranged = len(rest) > 1 and rest[1] == "true"
        accum = len(rest) > 2 and rest[2] == "true"
        views = len(rest) > 3 and rest[3] == "true"
    else:      # <K, kSpread, kPacket, kAllNodes, kSpheres[, kRays[, kAnyHit[, kMultiHit]]]>, false when absent
        rays, any_hit, multi_hit = [a == "true" for a in rest] + [False] * (3 - len(rest))
        kind = KINDS[0 if not rays else 2 if any_hit else 3 if multi_hit else 1]
    return (f"render_warpqueue_kernel[K={k}, spread={spread}, packet={packet}, all_nodes={all_nodes}, spheres={spheres}, "
            f"query={kind}{', ranged' if ranged else ''}{', accum' if accum else ''}{', views' if views else ''}]")


def main():
    old, new = ({(canonical(n), i): b for (n, i), b in functions(path).items()} for path in sys.argv[1:3])
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
