"""Search for ANI inputs where CUDA's double pow / exp and glibc's round differently (run once on a GPU machine).

The ANI gate (`final_ani < min_ani`) and the winner order (final_est_ani descending) turn a last-bit difference into a
different row set.  Random inputs never land there, so tests/ani_ties.py pins integer tuples found by this search:

  naive     (k, n, gl): ANI = pow(RN(n / gl), RN(1 / k))
  adjusted  (k, h1, h2, z): the hit counts {1: h1, 2: h2} (h1 > h2 >= 3, so mode 1 and lambda = RN(h2 / h1) * 2) and
            z unhit k-mers: ANI = pow(RN(RN(nz / RN(1 - RN(exp(-lambda)))) / nfull), RN(1 / k)), nz = h1 + h2,
            nfull = nz + z
  pairs     two adjusted tuples whose glibc ANIs are adjacent doubles

CUDA's values (torch float64 on the device) only choose the inputs: tuples where CUDA and glibc (Python's float
arithmetic, which calls glibc; numpy's own vectorised pow / exp is not glibc's on every CPU) disagree come first, so
the pinned tests fail on a device that rounds like CUDA's pow / exp.  Whether torch reaches the same libdevice pow as
the library is not checked here; the tests check the library's own rows.

    python scripts/find_ani_ties.py OUT.json
"""
import json
import math
import sys

import numpy as np
import torch


def naive(k):
    gl = np.repeat(np.arange(50, 3001, dtype=np.int64), np.arange(50, 3001))
    n = np.concatenate([np.arange(1, g + 1) for g in range(50, 3001)])
    x = n.astype(np.float64) / gl.astype(np.float64)
    c = 1.0 / k
    host = np.array([v ** c for v in x.tolist()])
    dev = torch.pow(torch.from_numpy(x).cuda(), torch.tensor(c, dtype=torch.float64, device="cuda")).cpu().numpy()
    bad = np.nonzero(host != dev)[0]
    return [dict(k=k, n=int(n[i]), gl=int(gl[i]), glibc=float(host[i]).hex(), cuda=float(dev[i]).hex()) for i in bad], len(x)


def adjusted_grid(h1_max, z_max):
    h1 = torch.arange(4, h1_max + 1, device="cuda", dtype=torch.int64)
    h2 = torch.arange(3, h1_max, device="cuda", dtype=torch.int64)
    H1, H2 = torch.meshgrid(h1, h2, indexing="ij")
    keep = (H2 < H1) & (H1 + H2 >= 25)
    H1, H2 = H1[keep], H2[keep]
    z = torch.arange(0, z_max + 1, device="cuda", dtype=torch.int64)
    return H1, H2, z


def adjusted_ani_dev(h1, h2, z, k):
    lam = h2.double() / h1.double() * 2.0
    nz = (h1 + h2).double()
    x1 = torch.exp(-lam)
    adj = nz / (1.0 - x1) / (nz + z.double())
    return torch.pow(adj, torch.tensor(1.0 / k, dtype=torch.float64, device="cuda"))


def adjusted_ani_host(h1, h2, z, k):
    c = 1.0 / k
    out = []
    for a, b, u in zip(*(np.asarray(t, dtype=np.float64).tolist() for t in (h1, h2, z))):
        nz = a + b
        out.append((nz / (1.0 - math.exp(-(b / a * 2.0))) / (nz + u)) ** c)
    return np.array(out)


def adjusted(k, h1_max=400, z_max=400, pair_cap=2000):
    H1, H2, z = adjusted_grid(h1_max, z_max)
    out, n_all = [], 0
    for zz in z.tolist():
        Z = torch.full_like(H1, zz)
        Z = torch.where(H1 + H2 + Z >= 50, Z, torch.full_like(Z, -1))
        m = Z >= 0
        h1, h2, Z = H1[m], H2[m], Z[m]
        dev = adjusted_ani_dev(h1, h2, Z, k).cpu().numpy()
        h1n, h2n, zn = h1.cpu().numpy(), h2.cpu().numpy(), Z.cpu().numpy()
        host = adjusted_ani_host(h1n, h2n, zn, k)
        n_all += len(dev)
        for i in np.nonzero(host != dev)[0][:20]:
            if len(out) < pair_cap:
                out.append(dict(k=k, h1=int(h1n[i]), h2=int(h2n[i]), z=int(zn[i]), glibc=float(host[i]).hex(), cuda=float(dev[i]).hex()))
    return out, n_all


def pairs(k, h1_max, z_max, cap=200):
    """adjacent-double pairs of glibc ANIs among the adjusted tuples; candidates by CUDA's values (within 4 ulp)"""
    H1, H2, z = adjusted_grid(h1_max, z_max)
    Z = z.repeat(len(H1))
    h1, h2 = H1.repeat_interleave(len(z)), H2.repeat_interleave(len(z))
    m = h1 + h2 + Z >= 50
    h1, h2, Z = h1[m], h2[m], Z[m]
    ani = adjusted_ani_dev(h1, h2, Z, k)
    ani, order = torch.sort(ani)
    bits = ani.view(torch.int64)
    gap = bits[1:] - bits[:-1]
    cand = torch.nonzero((gap >= 1) & (gap <= 4)).flatten()
    ia, ib = order[cand], order[cand + 1]
    A = [t[ia].cpu().numpy() for t in (h1, h2, Z)]
    B = [t[ib].cpu().numpy() for t in (h1, h2, Z)]
    ga, gb = adjusted_ani_host(*A, k), adjusted_ani_host(*B, k)
    ca, cb = ani[cand].cpu().numpy(), ani[cand + 1].cpu().numpy()
    out = []
    for i in range(len(cand)):
        lo, hi = sorted((ga[i], gb[i]))
        if np.nextafter(lo, np.inf) != hi:
            continue
        teeth = not ((ga[i] < gb[i]) == (ca[i] < cb[i]) and (ga[i] > gb[i]) == (ca[i] > cb[i]))
        out.append(dict(k=k, a=[int(A[0][i]), int(A[1][i]), int(A[2][i])], b=[int(B[0][i]), int(B[1][i]), int(B[2][i])],
                        glibc=[float(ga[i]).hex(), float(gb[i]).hex()], cuda=[float(ca[i]).hex(), float(cb[i]).hex()],
                        teeth=teeth))
    out.sort(key=lambda d: not d["teeth"])
    return out[:cap], int(len(h1))


def main():
    res = {"device": torch.cuda.get_device_name(0)}
    for k in (21, 31):
        bad, n = naive(k)
        res["naive_%d" % k] = dict(n=n, mismatches=len(bad), items=bad[:3000])
        bad, n = adjusted(k)
        res["adjusted_%d" % k] = dict(n=n, items=bad)
        p, n = pairs(k, 700, 600)
        res["pairs_%d" % k] = dict(n=n, items=p)
        print(k, res["naive_%d" % k]["mismatches"], "naive mismatches;", len(res["adjusted_%d" % k]["items"]),
              "adjusted;", len(p), "pairs,", sum(d["teeth"] for d in p), "with teeth", flush=True)
    with open(sys.argv[1], "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main()
