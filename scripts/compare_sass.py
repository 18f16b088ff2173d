"""Compares the sm_90a SASS of every kernel in two objects (cuobjdump -sass), instruction by instruction, with the
addresses stripped: which kernels a change left identical, which it changed, which it added.

    python scripts/compare_sass.py old/crt_cuda_core.o chameleonrt_b200/csrc/crt_cuda_core.o ['regex of kernel names']
"""
import re, subprocess, sys
def funcs(path):
    out = subprocess.check_output(["/usr/local/cuda/bin/cuobjdump", "-sass", path], text=True)
    res, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1); res[cur] = []; continue
        if cur and line.strip().startswith("/*"):
            res[cur].append(re.sub(r"^\s*/\*[0-9a-f]{4}\*/", "", line).strip())
    return res
a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
pat = re.compile(sys.argv[3]) if len(sys.argv) > 3 else None
same = diff = 0
for k in sorted(a):
    if pat and not pat.search(k): continue
    if k not in b: print("MISSING in new:", k); diff += 1; continue
    if a[k] == b[k]: same += 1
    else: print("DIFFERS:", k, len(a[k]), len(b[k])); diff += 1
print(f"identical {same}, differ {diff}; new-only: {sorted(set(b) - set(a))}")
