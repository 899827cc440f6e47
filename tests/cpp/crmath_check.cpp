// Host build of crmath.cuh.
//
// `crmath_check sweep N`: against libquadmath (113-bit powq / expq) on N inputs of each shape the ANI takes
//   naive     pow(RN(n / gl), RN(1 / k))
//   exp       exp(-lambda), lambda = RN(RN(cp1 / cm) * (mode + 1))
//   adjusted  pow(RN(RN(nz / RN(1 - RN(exp(-lambda)))) / nfull), RN(1 / k))
// for k = 21 and 31, each refined from libm's result moved by -2..+2 ulp (CUDA's pow is within 2 ulp).  Prints one
// line per shape: inputs, refinements != the rounded quad value, libm != it (the host libm's own misroundings), and
// inputs the quad value cannot decide (within 2^-100 of a rounding midpoint).
// `crmath_check eval`: reads "pow X C" / "exp Z" lines (hex doubles) and prints cr_pow / cr_exp of each in hex.
#include <quadmath.h>

#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "crmath.cuh"

static uint64_t rng_state = 0x5eed5eed12345678ull;
static uint64_t next_u64() {  // splitmix64
    uint64_t z = (rng_state += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
static uint64_t uniform(uint64_t lo, uint64_t hi) { return lo + next_u64() % (hi - lo + 1); }

struct Tally { long n = 0, cr_bad = 0, libm_bad = 0, undecided = 0; };

// the double nearest q, or false when q lies within 2^-100 (relative) of a midpoint between two doubles
static bool round_quad(__float128 q, double *out) {
    const double y = (double)q;
    const double up = nextafter(y, INFINITY), dn = nextafter(y, 0.);
    const __float128 mid_up = ((__float128)y + (__float128)up) / 2, mid_dn = ((__float128)y + (__float128)dn) / 2;
    const __float128 tol = q * (__float128)0x1p-100;
    *out = y;
    return fabsq(q - mid_up) > tol && fabsq(q - mid_dn) > tol;
}

static double step(double y, int j) {
    for (; j > 0; j--) y = nextafter(y, INFINITY);
    for (; j < 0; j++) y = nextafter(y, 0.);
    return y;
}

// every refinement of y0 moved by -2..+2 ulp must give the correctly rounded value
template <class F>
static void check(Tally &t, double want_cr, bool decided, double libm, F refine) {
    t.n++;
    if (!decided) { t.undecided++; return; }
    bool bad = false;
    for (int j = -2; j <= 2; j++) bad |= refine(step(libm, j)) != want_cr;
    t.cr_bad += bad;
    t.libm_bad += libm != want_cr;
}

static int eval() {
    char op[8];
    double a, b;
    while (scanf("%7s %la", op, &a) == 2) {
        if (!strcmp(op, "pow")) {
            if (scanf("%la", &b) != 1) return 1;
            printf("%a\n", crm::cr_pow(a, b));
        } else {
            printf("%a\n", crm::cr_exp(a));
        }
    }
    return 0;
}

int main(int argc, char **argv) {
    if (argc > 1 && !strcmp(argv[1], "eval")) return eval();
    const long N = argc > 2 ? atol(argv[2]) : 1000000;
    Tally naive, ex, adj;
    for (long i = 0; i < N; i++) {
        const int k = (i & 1) ? 31 : 21;
        const double c = 1. / k;
        // naive: gl up to 2^24 genome k-mers, n hits
        {
            const uint64_t gl = uniform(50, i % 3 == 0 ? 5000 : (1u << 24)), n = uniform(1, gl);
            const double x = (double)n / (double)gl;
            double want;
            const bool ok = round_quad(powq((__float128)x, (__float128)c), &want);
            check(naive, want, ok, pow(x, c), [&](double y0) { return crm::pow_refine(x, c, y0); });
        }
        // exp and adjusted: a ratio_lambda value and the counts around it
        {
            const uint64_t cm = uniform(3, i % 3 == 0 ? 200 : 100000), cp1 = uniform(3, cm), mode = uniform(1, 15);
            const double lam = (double)cp1 / (double)cm * (double)(mode + 1);
            double want;
            bool ok = round_quad(expq(-(__float128)lam), &want);
            check(ex, want, ok, exp(-lam), [&](double y0) { return crm::exp_refine(-lam, y0); });
            const uint64_t nfull = uniform(50, 1u << 24), nz = uniform(1, nfull);
            const double x = (double)nz / (1. - crm::cr_exp(-lam)) / (double)nfull;
            ok = round_quad(powq((__float128)x, (__float128)c), &want);
            check(adj, want, ok, pow(x, c), [&](double y0) { return crm::pow_refine(x, c, y0); });
        }
    }
    const char *names[3] = {"naive", "exp", "adjusted"};
    const Tally *ts[3] = {&naive, &ex, &adj};
    for (int s = 0; s < 3; s++)
        printf("tally %s n=%ld cr_bad=%ld libm_bad=%ld undecided=%ld\n", names[s], ts[s]->n, ts[s]->cr_bad, ts[s]->libm_bad,
               ts[s]->undecided);
    return 0;
}
