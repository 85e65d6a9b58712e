#!/bin/bash
# Whole-library SASS evidence (run on the CPU box): per sm_90a kernel the counts of the Hopper mnemonics
# (HGMMA = wgmma.mma_async, UTMALDG = TMA load, SYNCS = mbarrier operations), of MUFU (ex2 of the softmax) and of
# local-memory traffic (LDL/STL: register spills), plus the library totals.  usage: tools/sass_summary.sh [lib.so]
LIB=${1:-perceiver_io_b200/lib/libpcv_attn.so}
cuobjdump -sass $LIB > /tmp/sass_all.txt
python3 - <<'PY'
import re, collections
cur=None; per=collections.OrderedDict()
keys=["HGMMA","UTMALDG","SYNCS","MUFU","LDL","STL"]
for line in open('/tmp/sass_all.txt'):
    m=re.search(r"Function : (\S+)", line)
    if m:
        cur=m.group(1); per[cur]=collections.Counter(); continue
    m=re.match(r"\s+/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_]+)", line)
    if m and cur:
        op=m.group(2)
        for k in keys:
            if op.startswith(k): per[cur][k]+=1
        per[cur]["total"]+=1
tot=collections.Counter()
print("| kernel | " + " | ".join(keys) + " | instructions |"); print("|---|" + "---|"*(len(keys)+1))
import subprocess
for fn,c in per.items():
    tot.update(c)
    if c["HGMMA"] or c["UTMALDG"] or c["total"]>1500:
        name=subprocess.run(["c++filt",fn],capture_output=True,text=True).stdout.strip()
        name=re.sub(r"pcv::\(anonymous namespace\)::","",name); name=re.sub(r"\(CUtensorMap_st.*","",name)[:70]
        print(f"| {name} | " + " | ".join(str(c[k]) for k in keys) + f" | {c['total']} |")
print(f"| **library total ({len(per)} kernels)** | " + " | ".join(str(tot[k]) for k in keys) + f" | {tot['total']} |")
PY
