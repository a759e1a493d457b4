#!/usr/bin/env python
"""Counts, per kernel of libwukong_b200.so, the SASS instructions that prove which data-movement hardware a kernel uses
(cuobjdump -sass, sm_90a): UBLKCP (cp.async.bulk, the TMA engine's 1-D copies), SYNCS (mbarrier), LDGSTS (cp.async),
ACQBULK (griddepcontrol.wait of programmatic dependent launch), ATOMG...SYS (remote reservations over NVLink), CCTL.IVALL (L1
invalidation of a gpu / system fence), MATCH.ANY (the warp-level owner grouping of the exchange), STG.E.128 (its 16-byte stores).  Writes the markdown table of profiles/sass_evidence.md to stdout."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "wukong_b200", "libwukong_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", txt)), capture_output=True, text=True).stdout.split("\n")
PAT = re.compile(r"\b(UBLKCP(?:\.\w+)*|UTMALDG(?:\.\w+)*|SYNCS(?:\.\w+)*|LDGSTS(?:\.\w+)*|ACQBULK|ATOMG(?:\.\w+)*\.SYS|CCTL\.IVALL|MATCH\.ANY|STG\.E\.128)\b")
counts = collections.OrderedDict()
cur, k = None, -1
for line in txt.split("\n"):
    m = re.search(r"Function : (\S+)", line)
    if m:
        k += 1
        cur = re.sub(r"^void ", "", names[k])
        cur = re.sub(r"\(.*$", "", cur).replace("wk::", "")
        counts.setdefault(cur, collections.Counter())
        continue
    if cur is None:
        continue
    m = PAT.search(line)
    if m:
        counts[cur][m.group(1)] += 1
print("# SASS evidence of the data-movement instructions in libwukong_b200.so (cuobjdump -sass, sm_90a)\n")
print("Regenerate: `python scripts/sass_evidence.py > profiles/sass_evidence.md`.  Kernels with none of these instructions are left out;")
print("the template instances of one kernel that show the same counts are folded into one row.\n")
print("| kernel | instruction | count |\n|---|---|---|")
folded = collections.OrderedDict()
for kname, c in sorted(counts.items()):
    if not c:
        continue
    base = re.sub(r"<.*>$", "<...>", kname) if kname.startswith(("step_kernel", "expand_heavy")) else kname
    key = (base, tuple(sorted(c.items())))
    folded.setdefault(key, []).append(kname)
for (base, items), ks in folded.items():
    label = base if len(ks) == 1 and "<...>" not in base else "%s (%d instances)" % (base, len(ks))
    if len(ks) == 1:
        label = ks[0]
    for ins, n in items:
        print("| %s | %s | %d |" % (label, ins, n))
