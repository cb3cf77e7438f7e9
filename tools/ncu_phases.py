import csv, subprocess, sys
rep = sys.argv[1]; top = int(sys.argv[2]) if len(sys.argv)>2 else 40
out = subprocess.run(['ncu','-i',rep,'--page','details'],capture_output=True,text=True).stdout
for line in out.splitlines():
    if any(k in line for k in ('Duration','Executed Ipc Active','Issue Slots Busy','Executed Instructions','Registers Per','Dynamic Shared','Achieved Occupancy','Theoretical Occ','Avg. Active Threads','Warp Cycles Per Issued','One or More Eligible','Block Limit Shared','Block Limit Reg','L1/TEX Hit','bank conflict','stalled')):
        print(line.rstrip()[:150])
src = subprocess.run(['ncu','-i',rep,'--page','source','--print-source','cuda,sass','--csv'],capture_output=True,text=True).stdout
rows = list(csv.reader(src.splitlines()))
cur=None; agg={}; hdr=None
for r in rows:
    if not r: continue
    if r[0]=='File Path': cur=r[1].split('/')[-1]; continue
    if r[0]=='Line No': hdr=r; continue
    if r[0].isdigit() and hdr:
        try: inst=int(r[7]); samp=int(r[6])
        except: continue
        a=agg.setdefault((cur,int(r[0])),[0,0,r[1]]); a[0]+=inst; a[1]+=samp
tot=sum(a[0] for a in agg.values()); tots=sum(a[1] for a in agg.values())
print('total inst (line-attributed)',tot,'samples',tots)
# phase buckets by line ranges for swb_render.cuh
for k,a in sorted(agg.items(), key=lambda kv:-kv[1][0])[:top]:
    print('%9d %5.1f%% samp %5.1f%%  %s:%d  %s'%(a[0],100*a[0]/tot,100*a[1]/max(tots,1),k[0],k[1],a[2][:95]))
print('--- buckets')
import os
import re
SRC=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'spriteworld_b200', 'csrc', 'swb_render.cuh')
marks=[('A',r'// ---- phase A'),('B_pre',r'// ---- phase B'),('B1',r'^    // B1$'),('B2',r'^    // B2$'),('bgfill',r'// background fill'),('C_pre',r'// ---- phase C'),('H',r'---- H pass'),('V',r'---- V pass'),('D',r'// ---- phase D')]
lines=open(SRC).read().split('\n')
starts=[]
for name,pat in marks:
    for n,l in enumerate(lines,1):
        if re.search(pat,l): starts.append((n,name)); break
starts.sort()
kstart=[n for n,l in enumerate(lines,1) if 'render_kernel(DevState' in l][0]
def bucket(f,l):
    if f!='swb_render.cuh': return f
    if l<kstart: return 'helpers'
    cur='setup'
    for n,name in starts:
        if l>=n: cur=name
    return cur
b={}
for (f,l),a in agg.items():
    k=bucket(f,l); b[k]=b.get(k,0)+a[0]
for k,v in sorted(b.items(), key=lambda kv:-kv[1]): print('%-10s %6.1f%%  %d'%(k,100*v/tot,v))
