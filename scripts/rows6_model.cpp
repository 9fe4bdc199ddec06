// CPU model of k_rows6 / k_pop6 (bitswap_b200/csrc/rows6_core.cuh): runs the same per-lane arithmetic (quantised 4-bin groups,
// one chain per lane over its 8 chunks, re-anchored every R6_ANCHOR_BINS bins at S > 1024), the row's lanes in a loop,
// against the exact function on random uniform-grid rows, and checks
//   (1) every emitted integer pmf == the exact function's, (2) dead bins really have P == 1, (3) the worst screening error
//   of a trusted bin is far inside the window, (4) the chunk-base / pop search reproduces a search of the full table.
// Build: g++ -O2 -std=c++17 -o rows6_model scripts/rows6_model.cpp -lm ; run: ./rows6_model [rows] [seed] [S]
// S = 0 (default): the mix of S = 1024 / 256 / 64 rows; S = 2048 or 4096: every row at that support (quantbits 11 / 12),
// with needle-sharp, wide (every bin live), off-grid-mean and out-of-range rows among them.
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

int main(int argc, char **argv) {
    long nrows = argc > 1 ? atol(argv[1]) : 20000;
    if (argc > 2) rng ^= (uint64_t)atol(argv[2]) * 0x9E3779B97F4A7C15ull;
    const int Sw = argc > 3 ? atoi(argv[3]) : 0;
    if (Sw != 0 && Sw != 2048 && Sw != 4096) { printf("S must be 0, 2048 or 4096\n"); return 1; }
    const int bits = 31;
    long fixbad = 0, maxsteps = 0;
    long mism = 0, deadbad = 0, popbad = 0, doubted = 0, bins = 0, evaluated = 0, notok = 0;
    double worst = 0;  // window units
    double worst_frac = 0, worst64 = 0;
    for (long it = 0; it < nrows; ++it) {
        int mode = it % 8;
        int S = Sw ? Sw : ((mode == 6) ? 256 : (mode == 7 ? 64 : 1024));
        int q = S == 4096 ? 12 : (S == 2048 ? 11 : (S == 1024 ? 10 : (S == 256 ? 8 : 6)));
        const bool wide_s = S > 1024;
        std::vector<double> e(S);
        double lo, hi;
        if (S == 256 && !Sw) { for (int k = 1; k <= 255; ++k) e[k - 1] = (((double)k - 127.5) / 127.5) - 1. / 255.; }
        else { lo = -6 - urand(); hi = 6 + urand(); double step = (hi - lo) / S; for (int k = 0; k < S - 1; ++k) e[k] = lo + (k + 1) * step; }
        e[S - 1] = 1e300;
        // meta as k_row_meta computes it
        R6RowMeta M; int n = S - 1;
        M.a = e[0]; M.d = (e[n - 1] - e[0]) / (double)(n - 1);
        double dev = 0, emax = 0;
        for (int k = 0; k < n; ++k) { dev = fmax(dev, fabs(e[k] - fma((double)k, M.d, M.a))); emax = fmax(emax, fabs(e[k])); }
        dev += emax * 2.3e-16; M.dev = dev; M.rsv = 0;
        float muf, scf;
        switch (mode) {
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
    return (mism || popbad || fixbad) ? 2 : 0;
}
