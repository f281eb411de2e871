// The chi^2 tables of the RAIM stage (include/gpsb200.h: gpsb200_raim_thresholds; DESIGN §11.1) and the test
// multipliers K_fa of the ARAIM stage (gpsb200_araim_kfa; DESIGN §11.2), on the host.
//
// P(a, x), the regularized lower incomplete gamma function, by its power series below x = a + 1 and as 1 - Q(a, x)
// from the continued fraction of Q above; the chi^2(d) CDF at t is P(d / 2, t / 2). The noncentral chi^2(d, lambda)
// CDF is the Poisson(lambda / 2) mixture of central ones with d + 2k degrees of freedom. Both thresholds come from
// bisection on a bracket found by doubling; every term of the mixture is positive, so small probabilities keep their
// relative precision.
#include <cmath>

#include "pvt.h"

namespace gpsb200 {
namespace pvt {

namespace {

constexpr double kEps = 1e-17;

// exp(a ln x - x - lgamma(a)), the common factor of the series and the continued fraction
double gamma_factor(double a, double x) { return std::exp(a * std::log(x) - x - std::lgamma(a)); }

// Q(a, x) for x >= a + 1: the continued fraction 1 / (x + 1 - a - 1 (1 - a) / (x + 3 - a - ...)), modified Lentz.
double upper_cf(double a, double x) {
    const double tiny = 1e-300;
    double b = x + 1.0 - a, c = 1.0 / tiny, d = 1.0 / b, h = d;
    for (int i = 1; i < 10000; i++) {
        const double an = -i * (i - a);
        b += 2.0;
        d = an * d + b;
        if (std::fabs(d) < tiny) d = tiny;
        c = b + an / c;
        if (std::fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (std::fabs(del - 1.0) < kEps) break;
    }
    return gamma_factor(a, x) * h;
}

// P(a, x) for x < a + 1: sum_n x^n / (a (a + 1) ... (a + n)).
double lower_series(double a, double x) {
    double term = 1.0 / a, sum = term;
    for (int n = 1; n < 10000; n++) {
        term *= x / (a + n);
        sum += term;
        if (term < sum * kEps) break;
    }
    return gamma_factor(a, x) * sum;
}

double gamma_p(double a, double x) {
    if (x <= 0.0) return 0.0;
    return x < a + 1.0 ? lower_series(a, x) : 1.0 - upper_cf(a, x);
}

double gamma_q(double a, double x) {
    if (x <= 0.0) return 1.0;
    return x < a + 1.0 ? 1.0 - lower_series(a, x) : upper_cf(a, x);
}

// P(chi^2(d, lambda) <= t)
double ncx2_cdf(double t, int d, double lambda) {
    const double mu = lambda / 2.0, x = t / 2.0;
    if (mu == 0.0) return gamma_p(d / 2.0, x);
    // Poisson weights to mu + 40 sqrt(mu) + 60: the rest weighs less than 1e-100
    const int kmax = (int) (mu + 40.0 * std::sqrt(mu) + 60.0);
    double sum = 0.0;
    for (int k = 0; k <= kmax; k++) {
        const double w = std::exp(k * std::log(mu) - mu - std::lgamma(k + 1.0));
        sum += w * gamma_p(d / 2.0 + k, x);
    }
    return sum;
}

// The root of a decreasing f(v) - target on [0, inf): double the bracket, then bisect to the last representable step.
template <typename F> double solve_decreasing(F f, double target) {
    double lo = 0.0, hi = 1.0;
    while (f(hi) > target) {
        lo = hi;
        hi *= 2.0;
    }
    for (int i = 0; i < 200 && hi - lo > 1e-15 * hi; i++) {
        const double mid = 0.5 * (lo + hi);
        if (f(mid) > target) lo = mid;
        else hi = mid;
    }
    return 0.5 * (lo + hi);
}

// Q^-1(p) for 0 < p <= 0.5, Q the standard normal upper tail 0.5 erfc(x / sqrt 2): Newton on log Q(x) - log p from
// sqrt(-2 ln p), above the root (Q(x) <= exp(-x^2 / 2) / 2). log Q is concave and decreasing, so from above the steps
// approach the root monotonically and never overshoot.
double q_inv(double p) {
    const double lp = std::log(p);
    double x = std::sqrt(-2.0 * lp);
    for (int i = 0; i < 100; i++) {
        const double q = 0.5 * std::erfc(x / std::sqrt(2.0));
        const double phi = std::exp(-0.5 * x * x) / std::sqrt(2.0 * M_PI);
        const double dx = (std::log(q) - lp) * q / phi;
        x += dx;
        if (std::fabs(dx) <= 1e-16 * (1.0 + x)) break;
    }
    return x;
}

}  // namespace

bool araim_kfa(double p_fa_vert, double p_fa_horz, double *kh, double *kv) {
    if (!(p_fa_vert >= 1e-12 && p_fa_vert <= 0.5) || !(p_fa_horz >= 1e-12 && p_fa_horz <= 0.5)) return false;
    for (int n = 5; n < 5 + GPSB200_RAIM_MAX_DOF; n++) {
        kh[n - 5] = q_inv(p_fa_horz / (4.0 * n));
        kv[n - 5] = q_inv(p_fa_vert / (2.0 * n));
    }
    return true;
}

bool raim_thresholds(double p_fa, double p_md, double *T, double *lambda) {
    if (!(p_fa >= 1e-12 && p_fa <= 0.5) || !(p_md >= 1e-12 && p_md <= 0.5)) return false;
    for (int d = 1; d <= GPSB200_RAIM_MAX_DOF; d++) {
        const double t = solve_decreasing([d](double v) { return gamma_q(d / 2.0, v / 2.0); }, p_fa);
        T[d - 1] = t;
        lambda[d - 1] = solve_decreasing([d, t](double v) { return ncx2_cdf(t, d, v); }, p_md);
    }
    return true;
}

}  // namespace pvt
}  // namespace gpsb200
