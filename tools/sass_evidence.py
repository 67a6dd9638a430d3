#!/usr/bin/env python
"""tools/sass_evidence.py > profiles/<round>_sass_evidence.md — instruction mix per kernel of the in-tree liblmpc_b200.so
(cuobjdump -sass): the mnemonics that show what the kernels are built on (DMMA = fp64 tensor-core MMA, UBLKCP = 1-D bulk
async copy (TMA), REDUX/CREDUX = warp reductions, DFMA/DADD/DMUL = fp64 pipe, MUFU.RSQ64H/RCP64H = the approximations the custom
rsqrt / reciprocal refine) and what they are NOT (UTMALDG / HGMMA: no tiled TMA, no wgmma -- it has no fp64 type)."""
import collections, os, re, subprocess, sys
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(root, "racinglmpc_b200", "liblmpc_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", txt)))
kern = None; mix = collections.OrderedDict()
for line in txt.split("\n"):
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        mix[kern] = collections.Counter(); continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and kern:
        mix[kern][m.group(1)] += 1
keys = ["DMMA", "UBLKCP", "REDUX", "CREDUX", "DFMA", "DADD", "DMUL", "MUFU.RSQ64H", "MUFU.RCP64H", "SHFL", "LDS", "STS", "LDG", "BAR", "UTMALDG", "HGMMA"]
print("# SASS instruction mix of liblmpc_b200.so (static counts, `cuobjdump -sass`), arch %s\n" % ", ".join(arch))
print("| kernel | instructions | " + " | ".join(keys) + " |")
print("|---|---|" + "---|" * len(keys))
show = [k for k in mix if any(t in k for t in ("ftocp_kernel<12", "ftocp_kernel<14, 48", "ftocp_kernel<48, 0", "knn_ltv", "ss_select", "sim_step", "commit_laps_books", "pool_import", "probe_d"))]
for k in show:
    c = mix[k]
    tot = sum(c.values())
    def cnt(key):
        return sum(v for op, v in c.items() if op == key or op.startswith(key + "."))
    print("| `%s` | %d | " % (k.replace("lmpc::", ""), tot) + " | ".join(str(cnt(key)) for key in keys) + " |")
print("\n%d kernels in the library; every `ftocp_kernel<N,M>` instantiation has the same structure (DMMA sweeps, one UBLKCP staging)." % len(mix))
