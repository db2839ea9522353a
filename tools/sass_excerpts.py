"""Per kernel of libsige_b200.so, counts and first occurrences of the tensor-core / TMA / cluster SASS mnemonics
(which instructions the hot kernels really use).

    cuobjdump -sass sige_b200/lib/libsige_b200.so > sass.txt && python tools/sass_excerpts.py sass.txt
"""
import collections
import re
import sys

txt = open(sys.argv[1]).read()
funcs = re.split(r"\n\s*Function : ", txt)[1:]
print("# SASS evidence: cuobjdump -sass sige_b200/lib/libsige_b200.so (sm_90a), per kernel: instruction counts of the")
print("# tensor-core / TMA / cluster mnemonics and the first occurrence of each.\n")
pat = re.compile(r"\b(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UTMAPF|UBLKCP|SYNCS|HMMA|IMMA|LDSM|LDGSTS|UCGABAR|ACQBULK|ELECT|CCTL|REDG|STAS|MEMBAR|ERRBAR)(\.[A-Z0-9_.]+)?")
for f in funcs:
    name = f.split("\n", 1)[0].strip()
    if "sige" not in name:
        continue
    cnt, first, n_ins = collections.Counter(), {}, 0
    for ln in f.split("\n"):
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(.*?);", ln)
        if not m:
            continue
        n_ins += 1
        mm = pat.search(m.group(1))
        if mm:
            cnt[mm.group(1)] += 1
            first.setdefault(mm.group(1), m.group(1).strip())
    if not cnt:
        continue
    print("## %s" % name[:200])
    print("   %d SASS instructions; %s" % (n_ins, ", ".join("%s x%d" % kv for kv in cnt.most_common())))
    for k in ("UTCHMMA", "LDTM", "UTMALDG", "UBLKCP", "UTCBAR", "SYNCS", "HMMA", "LDSM", "STAS", "UCGABAR"):
        if k in first:
            print("      %-8s e.g.  %s" % (k, first[k][:150]))
    print()
