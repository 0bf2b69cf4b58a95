"""CPU statistics (NOT a measurement) of BASELINE config 4 -- two 500k x 500k R-MAT matrices,
16 nnz/row, C = A * B -- to see where the SpGEMM's products are: by nnz(C_i), by the length of
the A row and of the B rows streamed, and how full the 32-lane chunks of the column-panel
kernel are.  numpy regeneration of the same distribution (not the same seed as csrc/gen.cu).
It is the evidence behind the row routing in csrc/spgemm.cu."""
import numpy as np, sys
rng = np.random.default_rng(4)
SCALE, N, NPR = 19, 500_000, 16
a,b,c,d = .57,.19,.19,.05
def gen(seed, target):
    rng = np.random.default_rng(seed)
    M = int(target*1.35)
    rows = np.zeros(M, np.int64); cols = np.zeros(M, np.int64)
    for l in range(SCALE):
        u = rng.random(M)
        rbit = u >= a+b
        cbit = ((u >= a) & (u < a+b)) | (u >= a+b+c)
        rows = (rows<<1)|rbit; cols=(cols<<1)|cbit
    ok = (rows<N)&(cols<N)
    keys = np.unique((rows[ok]<<32)|cols[ok])
    if len(keys) > target:
        keys = np.sort(rng.choice(keys, target, replace=False))
    r = keys>>32; cc = keys & 0xffffffff
    ip = np.searchsorted(r, np.arange(N+1))
    return ip, cc
aip, aidx = gen(1, NPR*N)
bip, bidx = gen(2, NPR*N)
print("nnzA", len(aidx), "nnzB", len(bidx))
blen = np.diff(bip)
nprod = np.add.reduceat(np.concatenate([blen[aidx],[0]]), np.minimum(aip[:-1], len(aidx)))
nprod[np.diff(aip)==0] = 0
print("n_prod total %.3e"%nprod.sum(), "max row", nprod.max())
alen = np.diff(aip)
# sample rows weighted uniformly
S = 3000
samp = rng.choice(N, S, replace=False)
nnzc = np.zeros(S, np.int64)
for j,i in enumerate(samp):
    ks = aidx[aip[i]:aip[i+1]]
    if len(ks)==0: continue
    cols = np.concatenate([bidx[bip[k]:bip[k+1]] for k in ks])
    nnzc[j] = len(np.unique(cols))
np_s = nprod[samp]
print("est nnzC total %.3e" % (nnzc.mean()*N), "compression", np_s.sum()/max(nnzc.sum(),1))
for lo,hi in [(0,128),(128,1024),(1024,4096),(4096,16384),(16384,65536),(65536,10**9)]:
    m = (nnzc>lo)&(nnzc<=hi)
    print(f"nnzC in ({lo},{hi}]: rows {m.mean():.3f}  share of n_prod {np_s[m].sum()/np_s.sum():.3f}  share of nnzC {nnzc[m].sum()/nnzc.sum():.3f}  mean A len {alen[samp][m].mean() if m.any() else 0:.1f}")
print("B row length percentiles", np.percentile(blen,[50,90,99,99.9,100]))
# share of n_prod by B-row length (which B rows are streamed)
w = np.bincount(aidx, minlength=N)  # times each B row is used
tot = (w*blen).sum()
for lo,hi in [(0,32),(32,256),(256,2048),(2048,16384),(16384,10**9)]:
    m=(blen>lo)&(blen<=hi)
    print(f"B rows len ({lo},{hi}]: count {m.sum()} share of n_prod {(w*blen)[m].sum()/tot:.3f}")
print("---- by A row length")
for lo,hi in [(0,8),(8,64),(64,512),(512,4096),(4096,10**9)]:
    m=(alen>lo)&(alen<=hi)
    print(f"A len ({lo},{hi}]: rows {m.sum()} share n_prod {nprod[m].sum()/nprod.sum():.3f}")
# panel probes: for large rows (nnzC>4096 among sample), count (A nnz, panel) pairs with >=1 element and elements per pair
W=20480
P=(N+W-1)//W
big = samp[nnzc>4096]
pairs_nonempty=0; pairs_total=0; elems=0; iters=0
for i in big[:400]:
    ks = aidx[aip[i]:aip[i+1]]
    for k in ks:
        cols = bidx[bip[k]:bip[k+1]]
        cnt = np.bincount(cols//W, minlength=P)
        pairs_total += P; pairs_nonempty += (cnt>0).sum(); elems += cnt.sum(); iters += ((cnt+31)//32).sum() + (cnt%32==0).sum()*0
print("panel pairs total", pairs_total, "nonempty", pairs_nonempty, "elems", elems, "elems/nonempty pair %.1f"%(elems/pairs_nonempty), "lane efficiency %.2f"%(elems/(32*iters)))
