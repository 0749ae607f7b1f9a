"""Count Hopper tensor / async-copy SASS mnemonics per kernel of the built library (CPU-only evidence of what the
kernels are made of).  Usage: cuobjdump -sass llamagen_b200/lib/libllamagen_b200.so | python tools/sass_summary.py"""
import collections
import re
import subprocess
import sys

KEYS = ("HGMMA", "UTMALDG", "UBLKPF", "HMMA", "LDSM", "LDGSTS", "SYNCS", "ELECT", "ATOMS", "ATOMG", "ATOM.", "RED.", "REDUX")
counts = collections.defaultdict(collections.Counter)
cur = None
for line in sys.stdin:
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        continue
    if cur is None:
        continue
    m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m:
        for k in KEYS:
            if m.group(1).startswith(k):
                counts[cur][k] += 1


def demangle(n):
    try:
        d = subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    except Exception:
        d = n
    return re.sub(r"\(anonymous namespace\)::", "", d).split("(")[0][:100]


print("# cuobjdump -sass of the in-tree library: occurrences of selected mnemonics per kernel")
print("# HGMMA = wgmma   UTMALDG = TMA tensor load   UBLKPF = cp.async.bulk.prefetch.L2")
print("# HMMA = mma.sync   LDSM = ldmatrix   LDGSTS = cp.async   SYNCS = mbarrier ops   ATOMS = shared-memory atomics (")
print("# integer histogram counters of the sampler)   ATOMG / ATOM. / RED. = global atomics: only integer control counters (arrival ticket of sample_kernel's fused tail); no float atomics, none on a data path")
rows = sorted((demangle(fn), dict(c)) for fn, c in counts.items() if c)
for d, c in rows:
    print(f"{d}: {c}")
