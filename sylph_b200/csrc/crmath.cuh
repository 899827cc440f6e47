// crmath.cuh — correctly rounded pow and exp for positive finite doubles, host and device.
//
// CUDA's double pow (2 ulp) and exp (1 ulp) are not correctly rounded, and glibc's (0.52 ulp) are not either, but they
// round differently: an ANI one ulp off can fall on the other side of the -m gate or of another genome's ANI in the
// winner order.  cr_pow / cr_exp keep the library's result y0 (within a few ulp of the exact value) and move it to the
// double nearest the exact value: the offset of x^c (or e^z) from y0 is estimated in double-double from
// c*log(x) - log(y0) (or z - log(y0)), with log in double-double accurate to about 2^-95 absolute, and y0 steps to
// the neighbour that offset falls closest to.  An exact value within about 2^-35 ulp of a rounding midpoint cannot be
// decided at this precision; the nearer neighbour by the estimate is taken there (no such input among the 3 x 10^6
// that tests/cpp/crmath_check.cpp compares with 113-bit results, each refined from five starting values).
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define CRM_HD __host__ __device__ __forceinline__
#else
#define CRM_HD inline
#endif

namespace crm {

struct dd { double hi, lo; };

// a product that the compiler may not fuse into a later addition: the error-free transforms below take a rounded
// product p and its error fma(a, b, -p) apart, and an add of p contracted into an fma (nvcc does so across inlined
// calls) would pair an unrounded sum with the rounded p's error term
CRM_HD double mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

CRM_HD dd fast_two_sum(double a, double b) {  // |a| >= |b| or a == 0
    const double s = a + b;
    return {s, b - (s - a)};
}
CRM_HD dd two_sum(double a, double b) {
    const double s = a + b, bb = s - a;
    return {s, (a - (s - bb)) + (b - bb)};
}
CRM_HD dd dd_add(dd a, dd b) {
    dd s = two_sum(a.hi, b.hi);
    const dd t = two_sum(a.lo, b.lo);
    s = fast_two_sum(s.hi, s.lo + t.hi);
    return fast_two_sum(s.hi, s.lo + t.lo);
}
CRM_HD dd dd_neg(dd a) { return {-a.hi, -a.lo}; }
CRM_HD dd dd_mul(dd a, dd b) {
    const double p = mul(a.hi, b.hi);
    return fast_two_sum(p, fma(a.hi, b.hi, -p) + (a.hi * b.lo + a.lo * b.hi));
}
CRM_HD dd dd_mul_d(dd a, double b) {
    const double p = mul(a.hi, b);
    return fast_two_sum(p, fma(a.hi, b, -p) + a.lo * b);
}

// log(1 + j/128), j = 0..127, as hi + lo (hi = the double nearest, lo = the double nearest the rest)
#define CRM_LOG_TAB { \
    0x0.0p+0, 0x0.0p+0, 0x1.fe02a6b106789p-8, -0x1.e44b7e3711ebfp-67, \
    0x1.fc0a8b0fc03e4p-7, -0x1.83092c59642a1p-62, 0x1.7b91b07d5b11bp-6, -0x1.5b602ace3a510p-60, \
    0x1.f829b0e783300p-6, 0x1.33e3f04f1ef23p-60, 0x1.39e87b9febd60p-5, -0x1.5bfa937f551bbp-59, \
    0x1.77458f632dcfcp-5, 0x1.18d3ca87b9296p-59, 0x1.b42dd711971bfp-5, -0x1.eb9759c130499p-60, \
    0x1.f0a30c01162a6p-5, 0x1.85f325c5bbacdp-59, 0x1.16536eea37ae1p-4, -0x1.79da3e8c22cdap-60, \
    0x1.341d7961bd1d1p-4, -0x1.b599f227becbbp-58, 0x1.51b073f06183fp-4, 0x1.a49e39a1a8be4p-58, \
    0x1.6f0d28ae56b4cp-4, -0x1.906d99184b992p-58, 0x1.8c345d6319b21p-4, -0x1.4a697ab3424a9p-61, \
    0x1.a926d3a4ad563p-4, 0x1.942f48aa70ea9p-58, 0x1.c5e548f5bc743p-4, 0x1.5d617ef8161b1p-60, \
    0x1.e27076e2af2e6p-4, -0x1.61578001e0162p-60, 0x1.fec9131dbeabbp-4, -0x1.5746b9981b36cp-58, \
    0x1.0d77e7cd08e59p-3, 0x1.9a5dc5e9030acp-57, 0x1.1b72ad52f67a0p-3, 0x1.483023472cd74p-58, \
    0x1.29552f81ff523p-3, 0x1.301771c407dbfp-57, 0x1.371fc201e8f74p-3, 0x1.de6cb62af18a0p-58, \
    0x1.44d2b6ccb7d1ep-3, 0x1.9f4f6543e1f88p-57, 0x1.526e5e3a1b438p-3, -0x1.746ff8a470d3ap-57, \
    0x1.5ff3070a793d4p-3, -0x1.bc60efafc6f6ep-58, 0x1.6d60fe719d21dp-3, -0x1.caae268ecd179p-57, \
    0x1.7ab890210d909p-3, 0x1.be36b2d6a0608p-59, 0x1.87fa06520c911p-3, -0x1.bf7fdbfa08d9ap-57, \
    0x1.9525a9cf456b4p-3, 0x1.d904c1d4e2e26p-57, 0x1.a23bc1fe2b563p-3, 0x1.93711b07a998cp-59, \
    0x1.af3c94e80bff3p-3, -0x1.398cff3641985p-58, 0x1.bc286742d8cd6p-3, 0x1.4fce744870f55p-58, \
    0x1.c8ff7c79a9a22p-3, -0x1.4f689f8434012p-57, 0x1.d5c216b4fbb91p-3, 0x1.6e443597e4d40p-57, \
    0x1.e27076e2af2e6p-3, -0x1.61578001e0162p-59, 0x1.ef0adcbdc5936p-3, 0x1.48637950dc20dp-57, \
    0x1.fb9186d5e3e2bp-3, -0x1.caaae64f21acbp-57, 0x1.0402594b4d041p-2, -0x1.28ec217a5022dp-57, \
    0x1.0a324e27390e3p-2, 0x1.7dcfde8061c03p-56, 0x1.1058bf9ae4ad5p-2, 0x1.89fa0ab4cb31dp-58, \
    0x1.1675cababa60ep-2, 0x1.ce63eab883717p-61, 0x1.1c898c16999fbp-2, -0x1.0e5c62aff1c44p-60, \
    0x1.22941fbcf7966p-2, -0x1.76f5eb09628afp-56, 0x1.2895a13de86a3p-2, 0x1.7ad24c13f040ep-56, \
    0x1.2e8e2bae11d31p-2, -0x1.8f4cdb95ebdf9p-56, 0x1.347dd9a987d55p-2, -0x1.4dd4c580919f8p-57, \
    0x1.3a64c556945eap-2, -0x1.c68651945f97cp-57, 0x1.404308686a7e4p-2, -0x1.0bcfb6082ce6dp-56, \
    0x1.4618bc21c5ec2p-2, 0x1.f42decdeccf1dp-56, 0x1.4be5f957778a1p-2, -0x1.259b35b04813dp-57, \
    0x1.51aad872df82dp-2, 0x1.3927ac19f55e3p-59, 0x1.5767717455a6cp-2, 0x1.526adb283660cp-56, \
    0x1.5d1bdbf5809cap-2, 0x1.4236383dc7fe1p-56, 0x1.62c82f2b9c795p-2, 0x1.7b7af915300e5p-57, \
    0x1.686c81e9b14afp-2, -0x1.ddea0f7f58e3dp-57, 0x1.6e08eaa2ba1e4p-2, -0x1.cfb1b39ca3a0fp-56, \
    0x1.739d7f6bbd007p-2, -0x1.8c76ceb014b04p-56, 0x1.792a55fdd47a2p-2, 0x1.f057691fe9ed7p-56, \
    0x1.7eaf83b82afc3p-2, 0x1.92ce979ed2950p-56, 0x1.842d1da1e8b17p-2, 0x1.24ec519784676p-56, \
    0x1.89a3386c1425bp-2, -0x1.29639dfbbf0fbp-56, 0x1.8f11e873662c7p-2, 0x1.f85da755a61a3p-56, \
    0x1.947941c2116fbp-2, -0x1.16cc8bae0bbe4p-56, 0x1.99d958117e08bp-2, -0x1.a2b6889dc3e72p-57, \
    0x1.9f323ecbf984cp-2, -0x1.a92e513217f5cp-59, 0x1.a484090e5bb0ap-2, 0x1.5fe535b875a75p-57, \
    0x1.a9cec9a9a084ap-2, -0x1.cadec02b436afp-56, 0x1.af1293247786bp-2, 0x1.133844a15dc28p-58, \
    0x1.b44f77bcc8f63p-2, -0x1.cd04495459c78p-56, 0x1.b9858969310fbp-2, 0x1.663ec53e23bc4p-56, \
    0x1.beb4d9da71b7cp-2, -0x1.0f3c590a887cap-59, 0x1.c3dd7a7cdad4dp-2, 0x1.cecf052dea69bp-56, \
    0x1.c8ff7c79a9a22p-2, -0x1.4f689f8434012p-56, 0x1.ce1af0b85f3ebp-2, 0x1.edf4af2ab4267p-56, \
    0x1.d32fe7e00ebd5p-2, 0x1.877b232fafa37p-56, 0x1.d83e7258a2f3ep-2, 0x1.41456e8bb2511p-56, \
    0x1.dd46a04c1c4a1p-2, -0x1.0467656d8b892p-56, 0x1.e24881a7c6c26p-2, 0x1.cbd8f45954a46p-58, \
    0x1.e744261d68788p-2, -0x1.c825c90c344b9p-58, 0x1.ec399d2468cc0p-2, 0x1.75cee53f35397p-58, \
    0x1.f128f5faf06edp-2, -0x1.328df13bb38c3p-56, 0x1.f6123fa7028acp-2, 0x1.8515b0f2db341p-56, \
    0x1.faf588f78f31fp-2, -0x1.328260d8abca0p-57, 0x1.ffd2e0857f498p-2, 0x1.565f40d9321afp-56, \
    0x1.02552a5a5d0ffp-1, -0x1.cb1cb51408c00p-56, 0x1.04bdf9da926d2p-1, 0x1.97f304022c9dfp-55, \
    0x1.0723e5c1cdf40p-1, 0x1.395e58e2445bbp-55, 0x1.0986f4f573521p-1, -0x1.1b8095ac02f01p-55, \
    0x1.0be72e4252a83p-1, -0x1.259da11330801p-55, 0x1.0e44985d1cc8cp-1, -0x1.22a3442d2d384p-58, \
    0x1.109f39e2d4c97p-1, -0x1.0e09b27a4373ap-60, 0x1.12f719593efbcp-1, 0x1.4c048c671f435p-55, \
    0x1.154c3d2f4d5eap-1, -0x1.59c33171a6876p-55, 0x1.179eabbd899a1p-1, -0x1.00e7c6417e0b4p-55, \
    0x1.19ee6b467c96fp-1, -0x1.9d1a11443f10cp-56, 0x1.1c3b81f713c25p-1, -0x1.0dac1c4c810e9p-55, \
    0x1.1e85f5e7040d0p-1, 0x1.ef62cd2f9f1e3p-56, 0x1.20cdcd192ab6ep-1, -0x1.b2bf0bc229014p-55, \
    0x1.23130d7bebf43p-1, -0x1.f48725e374d6ep-55, 0x1.2555bce98f7cbp-1, 0x1.e021d6d6881e7p-56, \
    0x1.2795e1289b11bp-1, -0x1.487c0c246978ep-57, 0x1.29d37fec2b08bp-1, -0x1.bd1949a2d1982p-56, \
    0x1.2c0e9ed448e8cp-1, -0x1.1a158f3917586p-55, 0x1.2e47436e40268p-1, 0x1.0150861a4886bp-55, \
    0x1.307d7334f10bep-1, 0x1.fb590a1f566dap-57, 0x1.32b1339121d71p-1, 0x1.902ab5b3d916bp-56, \
    0x1.34e289d9ce1d3p-1, 0x1.6eb92d885ce4fp-57, 0x1.37117b54747b6p-1, -0x1.d117edbdd9103p-56, \
    0x1.393e0d3562a1ap-1, -0x1.58eef67f2483ap-55, 0x1.3b68449fffc23p-1, -0x1.41c484f9e9b26p-55, \
    0x1.3d9026a7156fbp-1, -0x1.6fef670bd4b62p-55, 0x1.3fb5b84d16f42p-1, 0x1.6d3a754172aefp-55, \
    0x1.41d8fe84672aep-1, 0x1.9192f30bd1806p-55, 0x1.43f9fe2f9ce67p-1, 0x1.e9c9ee6d83b86p-55, \
    0x1.4618bc21c5ec2p-1, 0x1.f42decdeccf1dp-55, 0x1.48353d1ea88dfp-1, 0x1.cf57a2ecc07f4p-55, \
    0x1.4a4f85db03ebbp-1, 0x1.13dfa3d3761b6p-60, 0x1.4c679afccee3ap-1, -0x1.3a5c4c8b39e41p-55, \
    0x1.4e7d811b75bb1p-1, -0x1.8d3d9ea6e9ea9p-55, 0x1.50913cc01686bp-1, 0x1.2f2ce96c2d5b1p-55, \
    0x1.52a2d265bc5abp-1, -0x1.1883750ea4d0ap-57, 0x1.54b2467999498p-1, -0x1.5baaf5d2f09f4p-55, \
    0x1.56bf9d5b3f399p-1, 0x1.0471885cd8ff3p-55, 0x1.58cadb5cd7989p-1, 0x1.849792ec98458p-56, \
    0x1.5ad404c359f2dp-1, -0x1.35955683f7196p-59, 0x1.5cdb1dc6c1765p-1, -0x1.cc2470e8a3df4p-55, \
    0x1.5ee02a9241675p-1, 0x1.c358257f49082p-55, 0x1.60e32f44788d9p-1, -0x1.ac1bb52fa589bp-56, \
}
#if defined(__CUDACC__)
__constant__ static const double log_tab_d[256] = CRM_LOG_TAB;
#endif
static const double log_tab_h[256] = CRM_LOG_TAB;
#undef CRM_LOG_TAB

// log(x) for a positive normal finite x, as a double-double (absolute error below 2^-95 for |log x| < 2^10):
// x = 2^e * m, m in [1, 2), m = t * (1 + s) / (1 - s) with t = 1 + j/128 the table point below m, |s| < 2^-8;
// log x = e*log 2 + log t + 2*atanh(s), the series in double-double up to s^3 and in double beyond.
CRM_HD dd log_dd(double x) {
#if defined(__CUDA_ARCH__)
    const double *tab = log_tab_d;
#else
    const double *tab = log_tab_h;
#endif
    int e;
    const double m = 2. * frexp(x, &e);  // exact
    e -= 1;
    const int j = (int)((m - 1.) * 128.);
    const double t = 1. + (double)j * (1. / 128.);
    const double num = m - t;              // exact: t <= m < 2t
    const dd den = two_sum(m, t);
    // s = num / den in double-double: one correction step of the quotient
    const double s1 = num / den.hi;
    const dd r = dd_add({num, 0.}, dd_mul_d(den, -s1));
    const dd s = fast_two_sum(s1, r.hi / den.hi);
    const dd s2 = dd_mul(s, s);
    const double z = s2.hi;
    const double tail = mul(z * z, 1. / 5. + z * (1. / 7. + z * (1. / 9. + z * (1. / 11.))));  // s^4/5 + ...
    // 2s * (1 + s^2/3 + tail)
    const dd third = {1. / 3., 0x1.5555555555555p-56};
    dd poly = dd_add(dd_mul(s2, third), {tail, 0.});
    poly = dd_add({1., 0.}, poly);
    dd l = dd_mul(dd_mul_d(s, 2.), poly);
    l = dd_add(l, {tab[2 * j], tab[2 * j + 1]});
    const dd ln2 = {0x1.62e42fefa39efp-1, 0x1.abc9e3b39803fp-56};
    return dd_add(l, dd_mul_d(ln2, (double)e));
}

// y0 ~ v: the double nearest v, given d ~ log(v / y0) (a few ulp at most)
CRM_HD double round_near(double y0, dd d) {
    // v - y0 = y0 * expm1(d), d tiny: y0 * (d + d^2/2)
    double off = y0 * (d.hi + (d.lo + 0.5 * d.hi * d.hi));
    double y = y0;
    for (int i = 0; i < 4; i++) {
        const double up = nextafter(y, INFINITY), dn = nextafter(y, 0.);
        if (off > 0.5 * (up - y)) { off -= up - y; y = up; }
        else if (off < -0.5 * (y - dn)) { off += y - dn; y = dn; }
        else break;
    }
    return y;
}

CRM_HD bool plain_positive(double v) { return v >= 2.2250738585072014e-308 && v <= 1.7976931348623157e308; }

// x^c rounded to nearest, from y0 = an approximation within 3 ulp; x > 0 (other inputs, and results outside the
// normal range, return y0)
CRM_HD double pow_refine(double x, double c, double y0) {
    if (!plain_positive(x) || !plain_positive(y0) || !(fabs(c) < 1e300)) return y0;
    return round_near(y0, dd_add(dd_mul_d(log_dd(x), c), dd_neg(log_dd(y0))));
}

// e^z rounded to nearest, from y0 = an approximation within 3 ulp (results outside the normal range return y0)
CRM_HD double exp_refine(double z, double y0) {
    if (!plain_positive(y0)) return y0;
    return round_near(y0, dd_add({z, 0.}, dd_neg(log_dd(y0))));
}

CRM_HD double cr_pow(double x, double c) { return pow_refine(x, c, pow(x, c)); }
CRM_HD double cr_exp(double z) { return exp_refine(z, exp(z)); }

}  // namespace crm
