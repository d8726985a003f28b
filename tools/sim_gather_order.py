#!/usr/bin/env python
"""CPU model of what a warp-wide gather touches under different particle orders of the counting sort.

A jittered lattice at the usual spacing h/2 is sorted (a) by h-cell, z fastest, then particle id (the engine's default), (b) with the cells split
in z (experiment K), (c) in "row order" (x / y binned at h/2, SALVA_B200_XYSUB=2).  Every particle's contact list is its neighbours within h in
ascending sorted index, as k_neighbors writes them; for every interior warp of 32 consecutive particles and every list position k the script
counts the distinct 32-byte sectors / 128-byte lines the k-th contacts of the 32 lanes fall into (records of 16 bytes), and the same per
quarter-warp (8 lanes), which is what the L1TEX data stage appears to pay for.  The last table splits each list over n lanes (the split
gather passes measured and not adopted, DESIGN.md 4a.15): a warp holds 32 / n particles, and in gather t lane u of particle p reads entry u + n t of p's list;
counts are per 32 contacts gathered.   usage: sim_gather_order.py [jitter amplitude in r, default 0.05]"""
import numpy as np, sys
from scipy.spatial import cKDTree
rng=np.random.default_rng(0)
r=0.025; h=4*r; nx,ny,nz=18,18,128
amp=float(sys.argv[1]) if len(sys.argv)>1 else 0.05
X,Y,Z=np.meshgrid(np.arange(nx),np.arange(ny),np.arange(nz),indexing='ij')
P=np.stack([X,Y,Z],-1).reshape(-1,3)*2*r + r
P=P+rng.uniform(-amp*r,amp*r,P.shape)
gid=np.arange(len(P))
def order(mode):
    c=np.floor(P/h).astype(int)
    if mode=='h': key=(c[:,0]*1000+c[:,1])*1000+c[:,2]
    elif mode=='rows':
        bx=np.floor(P[:,0]/(h/2)).astype(int); by=np.floor(P[:,1]/(h/2)).astype(int); key=(bx*1000+by)*1000+c[:,2]
    elif mode=='zsub2':
        bz=np.floor(P[:,2]/(h/2)).astype(int); key=(c[:,0]*1000+c[:,1])*1000+bz
    return np.lexsort((gid,key))
tree=cKDTree(P)
nb=tree.query_ball_point(P,h*(1+1e-9))
hi=np.array([nx,ny,nz])*2*r
for mode in ('h','zsub2','rows'):
    o=order(mode); rank=np.empty(len(P),int); rank[o]=np.arange(len(P))
    lists=[np.sort(rank[np.array(nb[i])]) for i in o]
    Q=P[o]
    inner=np.all((Q>3*h)&(Q<hi-3*h),axis=1)
    sect=[];lines=[];cnt=0
    for w0 in range(0,len(P)-31,32):
        if not inner[w0:w0+32].all(): continue
        L=[lists[s] for s in range(w0,w0+32)]
        M=max(len(x) for x in L)
        for k in range(M):
            js=np.array([x[k] for x in L if len(x)>k])
            sect.append(len(np.unique(js//2))*32/len(js)); lines.append(len(np.unique(js//8))*32/len(js))
        cnt+=1
    print("jitter %.2f r  %-6s warps %4d  mean contacts %.1f  sectors per 32-lane gather %.1f  128-byte lines %.1f"%(amp,mode,cnt,np.mean([len(x) for x,i in zip(lists,inner) if i]),np.mean(sect),np.mean(lines)))
print("---- quarter-warp model: sum over the 4 quarter-warps of distinct 128-byte lines / distinct 32-byte sectors")
for mode in ('h','rows'):
    o=order(mode); rank=np.empty(len(P),int); rank[o]=np.arange(len(P))
    lists=[np.sort(rank[np.array(nb[i])]) for i in o]
    Q=P[o]; inner=np.all((Q>3*h)&(Q<hi-3*h),axis=1)
    ql=[];qs=[]
    for w0 in range(0,len(P)-31,32):
        if not inner[w0:w0+32].all(): continue
        L=[lists[s] for s in range(w0,w0+32)]
        M=min(len(x) for x in L)
        for k in range(M):
            js=np.array([x[k] for x in L])
            ql.append(sum(len(np.unique(js[q*8:(q+1)*8]//8)) for q in range(4)))
            qs.append(sum(len(np.unique(js[q*8:(q+1)*8]//2)) for q in range(4)))
    print("jitter %.2f r  %-6s quarter-lines %.1f  quarter-sectors %.1f"%(amp,mode,np.mean(ql),np.mean(qs)))
print("---- lanes per particle (h order): per 32 contacts, distinct 32-byte sectors / 128-byte lines / quarter-warp 128-byte lines")
o=order('h'); rank=np.empty(len(P),int); rank[o]=np.arange(len(P))
lists=[np.sort(rank[np.array(nb[i])]) for i in o]
Q=P[o]; inner=np.all((Q>3*h)&(Q<hi-3*h),axis=1)
for n in (1,2,4,8):
    ps=32//n; sect=[];lines=[];ql=[]
    for w0 in range(0,len(P)-ps+1,ps):
        if not inner[w0:w0+ps].all(): continue
        L=[lists[s] for s in range(w0,w0+ps)]
        M=max(len(x) for x in L)
        for t in range((M+n-1)//n):
            js=np.array([L[l//n][l%n+n*t] if l%n+n*t<len(L[l//n]) else -1 for l in range(32)])  # lane l = (particle l // n, u = l % n)
            on=js>=0; k=on.sum(); a=js[on]
            sect.append(len(np.unique(a//2))*32/k); lines.append(len(np.unique(a//8))*32/k)
            ql.append(sum(len(np.unique(js[q*8:(q+1)*8][on[q*8:(q+1)*8]]//8)) for q in range(4))*32/k)
    print("jitter %.2f r  lanes %d (%2d particles per warp)  sectors %.1f  128-byte lines %.1f  quarter-warp lines %.1f"%(amp,n,ps,np.mean(sect),np.mean(lines),np.mean(ql)))
