"""CPU study: share of all gathers that target the k hottest labels (degree-sorted), RMAT EF16, and the same share
among the SELL rows' gathers alone (edges into rows of in-degree below the heavy threshold, 1024 by default; the
shared-memory table serves only those).  usage: topk_share.py <scale> [heavy_min_degree]"""
import sys, numpy as np
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
from memgraph_b200 import pagerank as pr
scale=int(sys.argv[1])
heavy_min=int(sys.argv[2]) if len(sys.argv) > 2 else 1024
n, m = 1<<scale, 16<<scale
s,t = pr.rmat_edges_host(scale, m)
indeg=np.bincount(t,minlength=n); outdeg=np.bincount(s,minlength=n)
order=np.lexsort((np.arange(n),-outdeg,-indeg))
pos=np.empty(n,dtype=np.int64); pos[order]=np.arange(n)
ps=pos[s]
ps_sell=ps[indeg[t] < heavy_min]
for k in (1,4,8,16,28,48,64,128,256,1024):
    print(f"scale {scale}: top {k}K labels receive {(ps < k*1024).mean():.3f} of the gathers, "
          f"{(ps_sell < k*1024).mean():.3f} of the SELL rows' ({len(ps_sell)} of {len(ps)})")
