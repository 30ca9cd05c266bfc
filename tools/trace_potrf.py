"""CVXB_TRACE timeline of one Cholesky inside the KKT factor (debug tool)."""
import os, sys, ctypes as C
os.environ["CVXB_TRACE"] = "1"
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cvxopt_b200, bench
from cvxopt_b200 import _lib
n = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
m = 2 * n
P, G, d, rng = bench.make_problem(n, m, 1)
k = cvxopt_b200.kkt_chol(G, {"l": m, "q": [], "s": []}, H=P)
W = {"d": d, "di": 1 / d, "v": [], "beta": [], "r": [], "rti": []}
for _ in range(3):
    k(W)
nb = (n + 127) // 128
full = np.zeros(8 * 4096, dtype=np.uint64)
_lib.load().cvxb_kkt_trace(k._h, full.ctypes.data, 4096)
buf = full[: nb * 8]
phr = full[8 * 2048:].reshape(-1, 8)[:nb].astype(np.float64)
ph = phr[:, :5]
t = buf.reshape(nb, 8).astype(np.float64)
t0 = t[0, 0]
t = np.where(t > 0, (t - t0) / 1e3, np.nan)
far = np.where(phr[:, 5:7] > 0, (phr[:, 5:7] - t0) / 1e3, np.nan)    # far update of the group ending at step j
print("breakdown", k.last_breakdown())
st = full[:nb*8].reshape(nb,8).astype(np.float64)
j = nb // 2
print("acc load+sync %.1f us" % ((ph[j,4]-ph[j,0])/1e3))
print("potf2 phases at step %d [us]: prologue-gemm1 %.1f | load+gemm2 %.1f | factor %.1f | inverse %.1f | store %.1f" % (j, (ph[j,0]-st[j,0])/1e3, (ph[j,1]-ph[j,0])/1e3, (ph[j,2]-ph[j,1])/1e3, (ph[j,3]-ph[j,2])/1e3, (st[j,1]-ph[j,3])/1e3))
print("step |  Dg start  end (dur) |  Tr start end | C0 start end | near start end | far start end   [us]")
for j in range(nb):
    r = t[j]
    print("%3d | %8.1f %8.1f (%5.1f) | %8.1f %8.1f | %8.1f %8.1f | %8.1f %8.1f | %8.1f %8.1f"
          % (j, r[0], r[1], r[1] - r[0], r[2], r[3], r[4], r[5], r[6], r[7], far[j, 0], far[j, 1]))
