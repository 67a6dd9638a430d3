#!/usr/bin/env python
"""tools/prof_report.py REPORT.ncu-rep MANGLED_KERNEL_PREFIX

Joins the SASS page of an `ncu --set full` report with `nvdisasm -g` line info of the in-tree liblmpc_b200.so and prints
(1) the headline raw metrics, (2) warp-stall samples / executed instructions / active threads per source region of
racinglmpc_b200/csrc/ftocp_pdip.cuh.  This is how the per-phase shares quoted in profiles/*.md were obtained.
Needs a writable /tmp/cub scratch directory."""
import os; os.makedirs("/tmp/cub", exist_ok=True)
import re, csv, collections, subprocess, sys, os
rep=sys.argv[1]; func=sys.argv[2]  # e.g. _Z12ftocp_kernelILi12ELi0ELi2ELi4ELb0EE
os.system('ncu -i %s --page raw --csv 2>/dev/null > /tmp/raw.csv'%rep)
os.system('ncu -i %s --page source --csv 2>/dev/null > /tmp/src.csv'%rep)
rows=list(csv.reader(open('/tmp/raw.csv'))); hdr=rows[0]; units=rows[1]; vals=rows[2]
keep=['gpu__time_duration.sum','dram__bytes_read.sum','dram__bytes_write.sum','launch__registers_per_thread','launch__shared_mem_per_block_dynamic','launch__occupancy_limit_registers','launch__occupancy_limit_shared_mem','sm__warps_active.avg.pct_of_peak_sustained_active','smsp__issue_active.avg.pct_of_peak_sustained_active','sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active','smsp__inst_executed.sum','smsp__thread_inst_executed_per_inst_executed.ratio','l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum','smsp__average_warp_latency_per_inst_issued.ratio']
summ={}
for i,h in enumerate(hdr):
    if h in keep or (h.startswith('smsp__average_warps_issue_stalled') and h.endswith('per_issue_active.ratio')):
        summ[h]=(vals[i],units[i])
for k in sorted(summ):
    try:
        if float(summ[k][0].replace(',',''))<0.05 and 'stalled' in k: continue
    except: pass
    print(k, summ[k])
os.system('cd /tmp/cub && rm -f *.cubin && cuobjdump -xelf all /root/repo/racinglmpc_b200/liblmpc_b200.so >/dev/null 2>&1 && nvdisasm -g -c *.cubin > all.sass 2>/dev/null')
lines=open('/tmp/cub/all.sass').read().split('\n')
start=[i for i,l in enumerate(lines) if l.startswith('.text.'+func)][0]
cur=None; insts=[]
for l in lines[start+1:]:
    if l.startswith('//---------------------'): break
    m=re.match(r'\s*//## File "([^"]+)", line (\d+)(.*)',l)
    if m: cur=(m.group(1).split('/')[-1], int(m.group(2))); continue
    m2=re.match(r'\s+/\*([0-9a-f]{4,})\*/\s+(.*?);',l)
    if m2: insts.append((cur, m2.group(2)))
rows=list(csv.reader(open('/tmp/src.csv'))); hdr=rows[1]; data=rows[2:]
print('insts',len(insts),'rows',len(data))
ci=hdr.index('# Samples'); ce=hdr.index('Instructions Executed'); ct=hdr.index('Thread Instructions Executed')
src=open('/root/repo/racinglmpc_b200/csrc/ftocp_pdip.cuh').read().split('\n')
# function ranges from source
marks=[(i+1,l.strip()) for i,l in enumerate(src) if 'static LMPC_HD' in l or '// ---- phase' in l or l.strip().startswith('// ---- ')]
def region(ln):
    r='?'
    for (n,t) in marks:
        if n<=ln: r=t[:60]
    return r
agg=collections.OrderedDict(); ops=collections.Counter()
n=min(len(insts),len(data))
for k in range(n):
    c=insts[k][0]
    key=region(c[1]) if c and c[0]=='ftocp_pdip.cuh' else ('other:'+(c[0] if c else '?'))
    a=agg.setdefault(key,[0,0,0]); a[0]+=int(data[k][ci]); a[1]+=int(data[k][ce]); a[2]+=int(data[k][ct])
    ops[insts[k][1].split()[0].split('.')[0]]+=int(data[k][ce])
tot=sum(a[0] for a in agg.values()); tote=sum(a[1] for a in agg.values())
for k,a in sorted(agg.items(), key=lambda kv:-kv[1][0]):
    if a[0]/tot>0.004: print('%5.1f%% smp %5.1f%% inst thr/inst %4.1f  %s'%(100*a[0]/tot,100*a[1]/tote,a[2]/max(a[1],1),k))
print(ops.most_common(14))
# top source lines (helps to split the '?' bucket = helpers above the first marked function)
byline=collections.defaultdict(lambda:[0,0])
for k in range(n):
    c=insts[k][0]
    if c and c[0]=='ftocp_pdip.cuh':
        byline[c[1]][0]+=int(data[k][ci]); byline[c[1]][1]+=int(data[k][ce])
print('top lines (line, %samples, %inst, text):')
for ln,(s_,e_) in sorted(byline.items(), key=lambda kv:-kv[1][0])[:int(os.environ.get('TOPLINES','25'))]:
    print('%5d %5.1f%% %5.1f%%  %s'%(ln,100*s_/tot,100*e_/tote,src[ln-1].strip()[:100]))
