// CPU model of k_rows6 / k_pop6 (bitswap_b200/csrc/rows6_core.cuh): runs the same per-lane arithmetic (quantised 4-bin groups,
// one chain per lane over its 8 chunks, re-anchored every R6_ANCHOR_BINS bins at S > 1024), the row's lanes in a loop,
// against the exact function on random uniform-grid rows, and checks
//   (1) every emitted integer pmf == the exact function's, (2) dead bins really have P == 1, (3) the worst screening error
//   of a trusted bin is far inside the window, (4) the chunk-base / pop search reproduces a search of the full table.
// Build: g++ -O2 -std=c++17 -o rows6_model scripts/rows6_model.cpp -lm ; run: ./rows6_model [rows] [seed] [S] [family]
// S = 0 (default): the mix of S = 1024 / 256 / 64 rows; S = 2048 or 4096: every row at that support (quantbits 11 / 12),
// with needle-sharp, wide (every bin live), off-grid-mean and out-of-range rows among them.
// family = 0 (default): every row spans about -6.5 .. 6.5.  1-6: the grids discretize() can build, np.linspace between the
// extrema of one latent dimension, with mu and sigma drawn relative to each grid (see grid_row):
//   1 off-centre (centre within +-1000, span 1-21)   2 float16 extrema at or near +-65504, possibly asymmetric
//   3 far from zero and narrow (30000-60000, span <= 1)   4 tiny spans 2^-20 .. 2^-24 at 0 and at 1000
//   5 coarse: dt = d / sigma just under and just over 64 (where the plan falls back)
//   6 rows perturbed off the affine line by up to the classification tolerance (windows up to the 262144 cap and past it)
// Rows that fail k_row_meta's rule get dev = +inf, as in the kernel (the plan then distrusts every bin).
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>
#include <string.h>
#include "../bitswap_b200/csrc/rows6_core.cuh"

static double rcp_fast(double d) {
    double y = r6_rcp_seed(d);
    double e = fma(-d, y, 1.0); e = fma(e, e, e); y = fma(y, e, y); e = fma(-d, y, 1.0);
    return fma(y, e, y);
}
static double cdf_fast(double e, double mu, double sc, double rsc) {      // host twin of bsw_cdf_fast
    double n = e - mu, q = n * rsc, rem = fma(-q, sc, n), t = fma(rem, rsc, q);
    if (t > 690.0) t = 690.0; if (t < -690.0) t = -690.0;
    return rcp_fast(1.0 + r6_exp_neg(t));
}
static double exact_pmf(const double *e, int k, int S, double m, double s, double rs) {
    double c = (k == S - 1) ? 1.0 : cdf_fast(e[k], m, s, rs);
    double p = (k == 0) ? 0.0 : cdf_fast(e[k - 1], m, s, rs);
    return c - p;
}
static uint64_t rng = 88172645463325252ull;
static double urand() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return (double)(rng >> 11) * (1.0 / 9007199254740992.0); }

constexpr int LPR = 4, CPL = 32 / LPR;      // the kernel's default mapping: 4 lanes per row, 8 chunks per lane

static double urange(double lo, double hi) { return lo + (hi - lo) * urand(); }
static double sgn() { return urand() < 0.5 ? -1.0 : 1.0; }
// round to the nearest float16 value (the samples discretize() takes the extrema of are float16), saturating at +-65504
static double half(double x) {
    if (x == 0.0) return 0.0;
    int ex; frexp(fabs(x), &ex);
    const int qe = std::max(ex - 11, -24);
    return fmax(-65504.0, fmin(65504.0, ldexp(nearbyint(ldexp(x, -qe)), qe)));
}

// One endpoint row of grid family fam (1-6) at support S as k_uniform_edges builds it (y_k = lo + k (hi - lo) / S, the
// multiply-add contracted), and mu / sigma drawn relative to the grid's centre c, half-width h and bin width d: a few bins
// live, many live, mass just beyond the grid, or anything in between.
static void grid_row(int fam, int S, std::vector<double> &e, float &muf, float &scf) {
    double lo, hi;
    switch (fam) {
        case 1: { const double c = urange(-1000, 1000), w = urange(1, 21); lo = half(c - w * urange(0.2, 0.8)); hi = half(lo + w); break; }
        case 2: { const int k = (int)(urand() * 4);
                  lo = k == 0 ? -65504.0 : half(-urange(30000, 65504));
                  hi = k == 1 ? 65504.0 : (k == 2 ? half(urange(-1000, 60000)) : half(urange(30000, 65504)));
                  if (k == 3) { lo = -65504.0; hi = 65504.0; }
                  break; }
        case 3: { const double c = sgn() * urange(30000, 60000), w = urange(1e-3, 1); lo = c - w * urange(0.2, 0.8); hi = lo + w; break; }
        case 4: { const double c = urand() < 0.5 ? 0.0 : 1000.0, w = ldexp(1.0, -20 - (int)(urand() * 5)); lo = c - w * urange(0.2, 0.8); hi = lo + w; break; }
        case 5: { lo = half(urange(-10, 5)); hi = half(lo + urange(0.5, 20)); break; }
        default: { lo = urange(-300, 300); hi = lo + exp(urange(log(0.5), log(100.0))); break; }
    }
    const double step = (hi - lo) / S;
    for (int k = 0; k < S - 1; ++k) e[k] = fma((double)(k + 1), step, lo);
    const double c = 0.5 * (lo + hi), h = 0.5 * (hi - lo), d = step;
    double mu, sc;
    if (fam == 5) {                                       // dt = d / sigma in 64 * [0.97, 1.03]
        sc = d / (64.0 * urange(0.97, 1.03)); mu = c + h * urange(-1, 1);
    } else {
        switch ((int)(urand() * 4)) {
            case 0: sc = d * pow(10.0, urange(-1.5, 0.5)); mu = c + h * urange(-1, 1); break;                  // a few bins live
            case 1: sc = h * urange(0.05, 0.6); mu = c + h * urange(-1, 1); break;                             // many live
            case 2: sc = d * pow(10.0, urange(-1, 1.5)); mu = c + sgn() * (h + sc * urange(0, 12)); break;     // just beyond the grid
            default: sc = d * pow(10.0, urange(0, log10(fmax(1.0, h / d)))); mu = c + h * urange(-1.2, 1.2); break;
        }
    }
    if (fam == 6) {                                       // deviation up to 1e-13 max(1, emax), the classification tolerance
        const double emax = fmax(fabs(lo), fabs(hi));
        const double dv = 1e-13 * fmax(1.0, emax) * pow(10.0, urange(-6, 0));
        for (int k = 1; k < S - 2; ++k) e[k] += dv * urange(-1, 1);
        e[1 + (int)(urand() * (S - 3))] += sgn() * dv;
    }
    muf = (float)mu; scf = (float)sc;
    if (!(scf > 0.0f)) scf = 1e-38f;
}

int main(int argc, char **argv) {
    long nrows = argc > 1 ? atol(argv[1]) : 20000;
    if (argc > 2) rng ^= (uint64_t)atol(argv[2]) * 0x9E3779B97F4A7C15ull;
    const int Sw = argc > 3 ? atoi(argv[3]) : 0;
    if (Sw != 0 && Sw != 2048 && Sw != 4096) { printf("S must be 0, 2048 or 4096\n"); return 1; }
    const int fam = argc > 4 ? atoi(argv[4]) : 0;
    if (fam < 0 || fam > 6) { printf("family must be 0 .. 6\n"); return 1; }
    const int bits = 31;
    long fixbad = 0, maxsteps = 0;
    long mism = 0, deadbad = 0, popbad = 0, doubted = 0, bins = 0, evaluated = 0, notok = 0, nonaffine = 0;
    double worst = 0;  // window units
    double worst_frac = 0, worst64 = 0;
    for (long it = 0; it < nrows; ++it) {
        int mode = it % 8;
        int S = Sw ? Sw : ((mode == 6) ? 256 : (mode == 7 ? 64 : 1024));
        int q = S == 4096 ? 12 : (S == 2048 ? 11 : (S == 1024 ? 10 : (S == 256 ? 8 : 6)));
        const bool wide_s = S > 1024;
        std::vector<double> e(S);
        double lo, hi;
        float muf, scf;
        if (fam) grid_row(fam, S, e, muf, scf);
        else if (S == 256 && !Sw) { for (int k = 1; k <= 255; ++k) e[k - 1] = (((double)k - 127.5) / 127.5) - 1. / 255.; }
        else { lo = -6 - urand(); hi = 6 + urand(); double step = (hi - lo) / S; for (int k = 0; k < S - 1; ++k) e[k] = lo + (k + 1) * step; }
        e[S - 1] = 1e300;
        // meta as k_row_meta computes it, classification included
        R6RowMeta M; int n = S - 1;
        M.a = e[0]; M.d = (e[n - 1] - e[0]) / (double)(n - 1);
        double dev = 0, emax = 0;
        for (int k = 0; k < n; ++k) { dev = fmax(dev, fabs(e[k] - fma((double)k, M.d, M.a))); emax = fmax(emax, fabs(e[k])); }
        dev += emax * 2.3e-16;
        const bool affine = (M.d > 0.0) && (dev <= 1e-13 * fmax(1.0, emax)) && (emax < 1e6);
        M.dev = affine ? dev : HUGE_VAL; M.rsv = 0;
        if (!affine) ++nonaffine;
        if (!fam) switch (mode) {
            case 0: case 1: muf = (float)((urand() - 0.5) * 10); scf = (float)(0.1 + 0.9 * urand()); break;
            case 2: muf = (float)((urand() - 0.5) * 14); scf = 0.1f + (float)(0.01 * urand()); break;             // sharp
            case 3: muf = (float)((urand() < 0.5 ? -1 : 1) * (7 + 20 * urand()));                                     // mass outside the grid,
                    scf = (it % 16 == 3) ? (float)((2. / 255.) / 8.) * (float)(1 + 30 * urand()) : (float)(0.1 + 0.9 * urand()); break;  // half of them needle-sharp (|t| >> 700 at the grid)
            case 4: muf = (float)((urand() - 0.5) * 4); scf = (float)(0.5 + 3 * urand()); break;                    // very wide
            case 5: muf = (float)((urand() - 0.5) * 12); scf = (float)(0.1 + 0.9 * urand()); break;
            case 6: if (Sw) { muf = (float)((urand() - 0.5) * 12); scf = (float)(1e-4 + 0.01 * urand()); break; }    // needle-sharp: a few bins live
                    muf = (float)((urand() - 0.5) * 2.4); scf = (urand() < 0.3) ? (float)((2. / 255.) / 8.) : (float)(0.00098 + 0.7 * urand() * urand()); break;
            default: if (Sw) { muf = (float)((urand() < 0.5 ? -1 : 1) * (30 + 1e4 * urand())); scf = (float)(0.1 + 0.9 * urand()); break; }  // far out of range
                     muf = (float)((urand() - 0.5) * 10); scf = (float)(0.1 + 0.9 * urand()); break;
        }
        double m = muf, s = scf, rs = 1.0 / s;
        double mult = (double)((1ll << bits) - (1ll << q)), mult2 = mult * 1048576.0;
        std::vector<uint32_t> Pex(S), P(S, 1u);
        for (int k = 0; k < S; ++k) Pex[k] = (uint32_t)(long long)(exact_pmf(e.data(), k, S, m, s, rs) * mult) + 1u;
        R6Plan pl = r6_plan(M, m, rs, S, bits);
        if (pl.mask == 0) ++notok;
        if (pl.kl % 4 || pl.kh % 4 || pl.kl < 0 || pl.kh > S || pl.kh <= pl.kl || pl.m < 4 || pl.m > (wide_s ? 128 : 32) || 32 * pl.m < pl.kh - pl.kl) { printf("bad plan kl %d kh %d m %d\n", pl.kl, pl.kh, pl.m); return 1; }
        // k_rows6's walk: LPR lanes share the row, lane j walks chunks j*CPL .. j*CPL+CPL-1 as ONE chain (anchored once)
        uint32_t lsum[32];
        for (int c = 0; c < 32; ++c) lsum[c] = 0;
        const double a = 1.0 / mult2, Tone = mult2 + R6_MAGIC0;
        const double rho1 = r6_exp_neg(pl.dt), rho4 = r6_exp_neg(4.0 * pl.dt);
        for (int j = 0; j < LPR; ++j) {
            const int ks0 = pl.kl + j * CPL * pl.m, kend = std::min(ks0 + CPL * pl.m, pl.kh);
            if (ks0 >= kend) continue;
            double ub = r6_exp_neg(fma((double)(ks0 - 1), pl.dt, pl.t0));
            double Tprev = ks0 == 0 ? R6_MAGIC0 : r6_quant(ub, a);
            long steps = 0;
            for (int k0 = ks0; k0 < kend; k0 += 4) {
                if (wide_s && k0 != ks0 && ((k0 - ks0) & (R6_ANCHOR_BINS - 1)) == 0) { ub = r6_exp_neg(fma((double)(k0 - 1), pl.dt, pl.t0)); steps = 0; }   // as r6_anchor
                maxsteps = std::max(maxsteps, ++steps);
                uint32_t dlo[4], dhi[4], vv[4];
                r6_group_q(ub, Tprev, rho1, rho4, a, Tone, k0 + 4 == S, {0, 0, 0, 0}, pl.win, dlo, dhi);
                bool any = false;
                for (int t = 0; t < 4; ++t) { vv[t] = r6_raw_q(dlo[t], dhi[t]) + 1u; any |= r6_doubt_q(dlo[t], pl.mask); }
                for (int t = 0; t < 4; ++t) {
                    ++evaluated;
                    if (pl.mask != 0 && !r6_doubt_q(dlo[t], pl.mask)) {
                        const double D = (double)(((uint64_t)dhi[t] << 32) | dlo[t]) - (double)pl.win;
                        double err = fabs(D - exact_pmf(e.data(), k0 + t, S, m, s, rs) * mult2);
                        worst = fmax(worst, err);
                        worst_frac = fmax(worst_frac, err / (double)pl.win);
                        if (pl.win == 64u) worst64 = fmax(worst64, err);
                    }
                }
                if (any)
                    for (int t = 0; t < 4; ++t) if (r6_doubt_q(dlo[t], pl.mask)) { vv[t] = (uint32_t)(long long)(exact_pmf(e.data(), k0 + t, S, m, s, rs) * mult) + 1u; ++doubted; }
                for (int t = 0; t < 4; ++t) { P[k0 + t] = vv[t]; lsum[(k0 + t - pl.kl) / pl.m] += vv[t]; }
            }
        }
        for (int k = 0; k < S; ++k) {
            ++bins;
            if (P[k] != Pex[k]) { ++mism; if (k < pl.kl || k >= pl.kh) ++deadbad; if (mism < 10) printf("mismatch row %ld mode %d k %d got %u want %u (kl %d kh %d m %d mu %g sc %g)\n", it, mode, k, P[k], Pex[k], pl.kl, pl.kh, pl.m, m, s); }
        }
        // remnant + bases + pop search vs a search of the full table
        uint64_t tot = 0; uint32_t best = 0; int bi = 0;
        for (int k = 0; k < S; ++k) { tot += Pex[k]; if (Pex[k] > best) { best = Pex[k]; bi = k; } }
        uint32_t rem = (uint32_t)((1ull << bits) - tot);
        if (wide_s) {                                     // the wide fix word round-trips (argmax, kl, kh, m)
            int b2, kl2, kh2, m2;
            r6_unfix_wide(r6_fix_wide(bi, pl.kl, pl.kh), b2, kl2, kh2, m2);
            if (b2 != bi || kl2 != pl.kl || kh2 != pl.kh || m2 != pl.m) ++fixbad;
        }
        std::vector<uint32_t> C(S + 1); C[0] = 0;
        for (int k = 0; k < S; ++k) C[k + 1] = C[k] + Pex[k] + (k == bi ? rem : 0);
        uint32_t base[32]; uint32_t acc = pl.kl;
        for (int lane = 0; lane < 32; ++lane) { int ks = pl.kl + lane * pl.m; base[lane] = acc + ((ks > bi) ? rem : 0); acc += lsum[lane]; }
        uint32_t Ckh = (1u << bits) - (uint32_t)(S - pl.kh);
        for (int trial = 0; trial < 8; ++trial) {
            uint32_t mm = trial == 0 ? 0 : (trial == 1 ? (1u << bits) - 1 : (uint32_t)(urand() * 2147483648.0));
            int want = (int)(std::upper_bound(C.begin(), C.begin() + S, mm) - C.begin()) - 1;
            int got;
            if (mm < (uint32_t)pl.kl) got = (int)mm;
            else if (mm >= Ckh) got = pl.kh + (int)(mm - Ckh);
            else {
                int chunk = -1; for (int l = 0; l < 32; ++l) if (base[l] <= mm) chunk = l;
                uint32_t cex = base[chunk]; got = -1;
                for (int l = 0; l < pl.m; ++l) { int k = pl.kl + chunk * pl.m + l; if (k >= pl.kh) break; if (cex <= mm) got = k; cex += P[k] + (k == bi ? rem : 0); }
            }
            if (got != want) { ++popbad; if (popbad < 10) printf("pop search row %ld mm %u got %d want %d (kl %d kh %d m %d bi %d)\n", it, mm, got, want, pl.kl, pl.kh, pl.m, bi); }
        }
    }
    printf("rows %ld bins %ld evaluated %ld (%.1f%%) exact-path %ld (%.4f%% of evaluated) plan-not-ok %ld\n", nrows, bins, evaluated, 100.0 * evaluated / bins, doubted, 100.0 * doubted / evaluated, notok);
    printf("worst trusted err among rows with the minimum window (64 units): %.2f units\n", worst64);
    printf("support %s: longest chain since its last exp %ld steps of 4 bins; wide fix-word mismatches %ld\n", Sw ? (Sw == 2048 ? "2048" : "4096") : "mixed", maxsteps, fixbad);
    printf("mismatches %ld (in dead zones %ld)  pop-search mismatches %ld  worst trusted err %.2f units (%.3f of its window)\n", mism, deadbad, popbad, worst, worst_frac);
    if (argc > 4) printf("family %d: rows not affine %ld\n", fam, nonaffine);
    return (mism || popbad || fixbad) ? 2 : 0;
}
