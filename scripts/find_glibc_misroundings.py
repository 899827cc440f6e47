"""Search for ANI inputs where glibc's pow / exp misround (CPU only; Python's float power and math.exp call glibc).

The device computes every ANI correctly rounded (sylph_b200/csrc/crmath.cuh); the reference calls glibc, whose pow is
0.52 ulp.  On the inputs this finds the two differ by one ulp, and tests/ani_ties.py pins them so that the device is
shown to keep the correctly rounded value where it matters:

  naive     (k, n, gl) with glibc's ANI one ulp from the correctly rounded one
  adjusted  (k, h1, h2, z), the spec of tests/ani_ties.py ({1: h1, 2: h2} hit counts, z unhit), likewise
  gate      a naive or adjusted input whose glibc ANI is the double below the correctly rounded one, and a -m percent p
            with RN(p / 100) == the correctly rounded ANI: correct rounding keeps the row, glibc drops it
  winner    adjusted specs A = (h1, h2, z) and B = (m h1, m h2, m z), whose ANIs are equal or adjacent doubles (the
            same rational, rounded along different paths), such that the profile winner of the k-mers they share differs
            between glibc and correct rounding in one genome order

The correctly rounded values come from Python decimal at 50 digits (oracle/pyref.py cr_pow / cr_exp).

    python scripts/find_glibc_misroundings.py [OUT.json]
"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import ani_ties as T  # noqa: E402


def naive(k, want, gl_max=3000):
    out = []
    for gl in range(50, gl_max + 1):
        for n in range(1, gl + 1, 7):
            if math.gcd(n, gl) != 1:
                continue
            spec = ("naive", n, gl)
            g = T.glibc_ani(spec, k)
            c = T.cr_ani(spec, k)
            if g != c:
                out.append(dict(k=k, spec=spec, glibc=g.hex(), cr=c.hex()))
                if len(out) >= want:
                    return out
    return out


def adj_specs(h1_max=200, z_max=400, step=13):
    for h1 in range(4, h1_max + 1):
        for h2 in range(3, h1):
            if h1 + h2 < 25:
                continue
            for z in range(0, z_max + 1, step):
                yield ("adj", h1, h2, z)


def adjusted(k, want):
    out = []
    for spec in adj_specs():
        g, c = T.glibc_ani(spec, k), T.cr_ani(spec, k)
        if g != c:
            out.append(dict(k=k, spec=spec, glibc=g.hex(), cr=c.hex()))
            if len(out) >= want:
                break
    return out


def gates(found):
    """inputs whose glibc ANI is the double below the correctly rounded one, with a percent mapping to the latter"""
    out = []
    for f in found:
        c, g = float.fromhex(f["cr"]), float.fromhex(f["glibc"])
        p = T.gate_percent(c)
        if g == math.nextafter(c, -math.inf) and p is not None and not g >= p / 100.0:
            out.append(dict(f, p=p.hex()))
    return out


def winner(a, b, ani):
    """the pass-2 winner of two genomes in this order: the greater ANI, the first on equal ANIs"""
    return a if ani[0] >= ani[1] else b


def winners(k, want, scales=(3, 5, 6, 7)):
    out = []
    for a in adj_specs(h1_max=120, step=7):
        for m in scales:
            b = ("adj", m * a[1], m * a[2], m * a[3])
            ga, gb = T.glibc_ani(a, k), T.glibc_ani(b, k)
            if abs(ga - gb) > 4 * (math.nextafter(ga, math.inf) - ga):
                continue
            ca, cb = T.cr_ani(a, k), T.cr_ani(b, k)
            if (ga, gb) == (ca, cb):
                continue
            for first, second, g, c in ((a, b, (ga, gb), (ca, cb)), (b, a, (gb, ga), (cb, ca))):
                if winner(0, 1, g) != winner(0, 1, c):
                    out.append(dict(k=k, a=first, b=second, glibc=[v.hex() for v in g], cr=[v.hex() for v in c]))
                    break
            if len(out) >= want:
                return out
    return out


def main():
    res = {}
    for k in (21, 31):
        res["naive_%d" % k] = naive(k, 6)
        res["adjusted_%d" % k] = adjusted(k, 6)
        res["gates_%d" % k] = gates(res["naive_%d" % k] + res["adjusted_%d" % k])
        res["winners_%d" % k] = winners(k, 2)
        print(k, {key: len(v) for key, v in res.items() if key.endswith(str(k))}, flush=True)
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(text)
    else:
        print(text)


if __name__ == "__main__":
    main()
