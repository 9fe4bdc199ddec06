// The direct-cdf coder (sm_90a): an opt-in quantiser with its own bitstreams (bsw_codec_set_coder, BSW_CODER_DIRECT).
//
// The reference quantiser (ANS.__init__, cifar_compress.py:28-39) couples every bin of a row: trunc(pmf * M) + 1, then the
// remnant 2^31 - sum goes to the row's argmax, so one integer cdf value needs the whole row.  The direct quantiser defines
// each integer cdf value from one float cdf value:
//
//     F_k = bsw_cdf_fast(e_k, mu, sigma)            k = 0 .. S-2  (a NaN argument counts as F = 0)
//     M'  = 2^31 - 2S
//     C_0 = 0,  C_S = 2^31,  C_k = floor(RN(F_{k-1} * M')) + 2k      k = 1 .. S-1
//     P_k = C_{k+1} - C_k
//
// The float cdf is accurate to a few ulps, far below 1/M', so where its evaluation is not monotone (nearly equal endpoints)
// the floor falls by at most 1 between neighbours; the margin of 2 per bin keeps every P_k >= 1 and C strictly increasing.
// P_0 and P_{S-1} are at least 2, and C_S is a constant: the +1e300 pad of an endpoint row is never evaluated.
//
// So a push needs C_s and C_{s+1}, and a pop the 32 chunk bases C_{j S/32} plus one chunk.  Two phases, as in ans_rows.cu:
//   phase A  k_direct_pairs: one thread per (stream, row) -> the (P_s, C_s, reciprocal) uint4 k_push_pairs reads
//            k_direct_bases: one thread per (stream, row, chunk) -> 32 chunk bases per row
//   phase B  k_push_pairs (ans_rows.cu, unchanged) / k_pop_direct: one warp per stream, ballot over the bases, then each
//            lane evaluates the upper cdf of one bin of the chosen chunk (S/1024 passes of 32 above 1024 bins)
// Every C_k, in every kernel, comes from direct_cdf() below, so encoder and decoder agree at any batch size and on any lane.
#include "coder.cuh"

namespace {

constexpr int DW = 4;        // warps per CTA of the serial pop, as k_pop_coarse

// C_k of the row starting at e (k = 0 .. S).  Explicit round-to-nearest intrinsics throughout, so no contraction can differ
// between the kernels that evaluate it.
__device__ __forceinline__ uint32_t direct_cdf(const double *__restrict__ e, int k, int S, double m, double s, double rs) {
    if (k <= 0) return 0u;
    if (k >= S) return 0x80000000u;
    const double ek = __ldg(e + k - 1);
    double F = bsw_cdf_fast(ek, m, s, rs);
    if (isnan(__dmul_rn(__dsub_rn(ek, m), rs))) F = 0.0;           // NaN mu or sigma (bsw_cdf_fast would clamp it to 1)
    const double Mp = (double)(0x80000000u - 2u * (uint32_t)S);
    return __double2uint_rz(__dmul_rn(F, Mp)) + 2u * (uint32_t)k;
}

// ---- phase A -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_direct_pairs(int count, int64_t L, const float *__restrict__ mu, int64_t mss,
        const float *__restrict__ sc, int64_t sss, const double *__restrict__ endp, int64_t ers,
        const int16_t *__restrict__ sym, int S, uint4 *__restrict__ pairs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)count * L) return;
    const int64_t si = i / L, row = i - si * L;
    const int sy = sym[i];
    if ((unsigned)sy >= (unsigned)S) { pairs[i] = make_uint4(0u, 0u, 0u, 0u); return; }     // flagged by k_push_pairs
    const double m = (double)mu[si * mss + row], s = (double)sc[si * sss + row];
    const double rs = __ddiv_rn(1.0, s);
    const double *e = endp + row * ers;
    const uint32_t c0 = direct_cdf(e, sy, S, m, s, rs), c1 = direct_cdf(e, sy + 1, S, m, s, rs);
    const uint32_t p = c1 - c0;
    const uint64_t M = ~0ull / (uint64_t)p;                          // reciprocal for the serial phase's division
    pairs[i] = make_uint4(p, c0, (uint32_t)M, (uint32_t)(M >> 32));
}

__global__ void __launch_bounds__(256) k_direct_bases(int count, int64_t L, const float *__restrict__ mu, int64_t mss,
        const float *__restrict__ sc, int64_t sss, const double *__restrict__ endp, int64_t ers, int S,
        uint32_t *__restrict__ bases) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)count * L * 32) return;
    const int64_t r = i >> 5, si = r / L, row = r - si * L;
    const double m = (double)mu[si * mss + row], s = (double)sc[si * sss + row];
    const double rs = __ddiv_rn(1.0, s);
    bases[i] = direct_cdf(endp + row * ers, (int)(i & 31) * (S / 32), S, m, s, rs);
}

// ---- phase B: pop --------------------------------------------------------------------------------------------------------
// Chunk j of a row holds the CH = S/32 bins [j CH, j CH + CH).  The chunk holding m = head & mask is the last one whose base
// is <= m; inside it, lane l evaluates the UPPER cdf C_{k+1} of bin k = k0 + l, and the symbol is the first bin whose upper
// cdf exceeds m.  Its lower cdf is the previous lane's value, or the carry (the chunk base, or the last upper cdf of the
// previous pass of 32 bins).  Below 1024 bins lanes >= CH idle; the chunk's last upper cdf is the next chunk's base, which is
// > m, so the last pass always finds the symbol.
// MASK: pixel level with block extents (bsw_x_live), as k_pop_coarse.
template <int NB, bool MASK>
__global__ void __launch_bounds__(DW * 32) k_pop_direct(bsw_streams sv, int first, int count, const float *__restrict__ mu,
        int64_t mss, const float *__restrict__ sc, int64_t sss, const double *__restrict__ endp, int64_t ers,
        const uint32_t *__restrict__ bases, int16_t *__restrict__ sym, int64_t L, const int16_t *__restrict__ ext) {
    constexpr int S = 32 * NB, CH = NB, NP = NB < 32 ? 1 : NB / 32;
    const int lane = threadIdx.x & 31;
    const int si = blockIdx.x * DW + (threadIdx.x >> 5);
    if (si >= count) return;
    const int b = first + si;
    WarpStream ws;
    ws.open(sv, b);
    if (ws.err) return;
    int vh = 32, vw = 32;
    if (MASK) { vh = ext[2 * si]; vw = ext[2 * si + 1]; }
    const float *mub = mu + (int64_t)si * mss, *scb = sc + (int64_t)si * sss;
    const uint32_t *cb = bases + (int64_t)si * L * 32;
    int16_t *sy = sym + (int64_t)si * L;
    const uint32_t mask = 0x7fffffffu;

    float mu_w = 0.f, sc_w = 1.f, mu_nx, sc_nx;
    int my_sym = 0;
    {
        int64_t r = ((L - 1) & ~(int64_t)31) + lane;
        mu_nx = r < L ? mub[r] : 0.f;
        sc_nx = r < L ? scb[r] : 1.f;
    }
    uint32_t base_n1 = __ldg(cb + (L - 1) * 32 + lane);
    uint32_t base_n2 = L > 1 ? __ldg(cb + (L - 2) * 32 + lane) : 0u;
    for (int64_t i = L - 1; i >= 0; --i) {
        const int j32 = (int)(i & 31);
        const bool new_block = (j32 == 31 || i == L - 1);
        if (new_block) { mu_w = mu_nx; sc_w = sc_nx; }
        const double m_ = (double)__shfl_sync(FULL, mu_w, j32), s_ = (double)__shfl_sync(FULL, sc_w, j32);
        if (new_block) {
            int64_t r = (i & ~(int64_t)31) - 32 + lane;
            mu_nx = r >= 0 ? mub[r] : 0.f;
            sc_nx = r >= 0 ? scb[r] : 1.f;
        }
        const uint32_t base = base_n1;
        base_n1 = base_n2;
        if (i > 1) base_n2 = __ldg(cb + (i - 2) * 32 + lane);
        if (!MASK || bsw_x_live(i, vh, vw)) {             // a masked dim leaves the head alone; its symbol is padded later
            const double rs = __ddiv_rn(1.0, s_);
            const uint32_t mm = (uint32_t)ws.x & mask;
            const int chunk = 31 - __clz(__ballot_sync(FULL, base <= mm));              // base 0 = C_0 <= mm always
            const double *e = endp + i * ers;
            uint32_t carry = __shfl_sync(FULL, base, chunk), ps = 1u, cs = 0u;
            int s = 0;
#pragma unroll 1
            for (int sub = 0; sub < NP; ++sub) {
                const int k0 = chunk * CH + sub * 32;
                const uint32_t up = lane < CH ? direct_cdf(e, k0 + lane + 1, S, m_, s_, rs) : 0xffffffffu;
                const uint32_t above = __ballot_sync(FULL, up > mm);
                if (above || sub == NP - 1) {
                    const int js = __ffs(above) - 1;
                    const uint32_t lo = __shfl_sync(FULL, up, (js - 1) & 31), hi = __shfl_sync(FULL, up, js & 31);
                    cs = js > 0 ? lo : carry;
                    ps = hi - cs;
                    s = k0 + js;
                    break;
                }
                carry = __shfl_sync(FULL, up, 31);
            }
            if (lane == j32) my_sym = s;
            ws.decode(ps, cs, mm, 31, lane);
        }
        if (j32 == 0 || ws.err) {                         // block of rows done: coalesced symbol store
            int64_t r = (i & ~(int64_t)31) + lane;
            if (r < L && r >= i) sy[r] = (int16_t)my_sym;
            if (ws.err) break;
        }
    }
    ws.close(sv, b, lane);
}

// ---- materialised tables (the shared prior and bsw_direct_tables) ---------------------------------------------------------
__global__ void k_direct_tables(const double *__restrict__ endp, int64_t ers, const double *__restrict__ mu,
        const double *__restrict__ sc, int64_t ms, int64_t L, int S, uint32_t *__restrict__ P, uint32_t *__restrict__ C) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L * S) return;
    const int64_t row = i / S;
    const int k = (int)(i - row * S);
    const double m = mu[row * ms], s = sc[row * ms];
    const double rs = __ddiv_rn(1.0, s);
    const double *e = endp + row * ers;
    const uint32_t c0 = direct_cdf(e, k, S, m, s, rs), c1 = direct_cdf(e, k + 1, S, m, s, rs);
    P[i] = c1 - c0;
    C[row * (S + 1) + k] = c0;
    if (k == S - 1) C[row * (S + 1) + S] = c1;
}

int direct_args_ok(bsw_streams *s, int first, int count, const float *mu, const float *sc, const double *endp, int64_t ers,
                   const int16_t *sym, int64_t L, int S, int bits, int q, const void *scratch) {
    BSW_REQUIRE(s && first >= 0 && count > 0 && first + count <= s->B, "direct coder: stream range out of bounds");
    BSW_REQUIRE(mu && sc && endp && sym && scratch && L > 0 && L < 65536 * 32, "direct coder: bad arguments");
    BSW_REQUIRE(bits == 31, "direct coder: bits must be 31 (the quantiser is defined for 2^31)");
    BSW_REQUIRE(q >= 0 && q < bits, "direct coder: quantbits out of range");
    BSW_REQUIRE(ers == 0 || ers >= S, "direct coder: endpoint rows must hold S doubles (+1e300 padded)");
    BSW_REQUIRE((((uintptr_t)scratch) & 15) == 0, "direct coder: scratch must be 16-byte aligned");
    return BSW_OK;
}

}  // namespace

// One phase of a direct level (phase 0 = the parallel kernel, 1 = the serial coder; both, in order, with the same scratch).
int bsw_direct_2p(int phase, bool pop, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc,
                  int64_t sss, const double *endp, int64_t ers, int16_t *sym, int64_t L, int S, void *scratch,
                  size_t scratch_bytes, const int16_t *ext, cudaStream_t st) {
    if (int rc = direct_args_ok(s, first, count, mu, sc, endp, ers, sym, L, S, 31, 0, scratch)) return rc;
    BSW_REQUIRE(scratch_bytes >= RowsScratch::bytes(pop, count, L), "direct coder: scratch too small");
    const RowsScratch scr(scratch, count, L);
    return with_support<1, 128>(S, "direct coder: support must be one of 32,64,...,4096", [&](auto nb) -> int {
        constexpr int NB = decltype(nb)::value;
        if (phase == 0) {
            const int64_t n = (int64_t)count * L * (pop ? 32 : 1);
            if (pop) k_direct_bases<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(count, L, mu, mss, sc, sss, endp, ers, S, scr.bases);
            else k_direct_pairs<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(count, L, mu, mss, sc, sss, endp, ers, sym, S, scr.pairs);
        } else {
            if (!pop) return bsw_push_pairs(s, first, count, scr.pairs, L, 31, ext, st);
            BSW_MAX_SHARED_ONCE((k_pop_direct<NB, false>)); BSW_MAX_SHARED_ONCE((k_pop_direct<NB, true>));
            const unsigned g = (count + DW - 1) / DW;
            if (ext) k_pop_direct<NB, true><<<g, DW * 32, 0, st>>>(*s, first, count, mu, mss, sc, sss, endp, ers, scr.bases, sym, L, ext);
            else k_pop_direct<NB, false><<<g, DW * 32, 0, st>>>(*s, first, count, mu, mss, sc, sss, endp, ers, scr.bases, sym, L, nullptr);
        }
        BSW_LAUNCH_CHECK();
        return BSW_OK;
    });
}

int bsw_direct_tables_st(const double *endp, int64_t ers, const double *mu, const double *sc, int64_t ms, int64_t L, int S,
                         uint32_t *P, uint32_t *C, cudaStream_t st) {
    BSW_REQUIRE(endp && mu && sc && P && C && L > 0, "bsw_direct_tables: bad arguments");
    BSW_REQUIRE(S >= 2 && S <= 4096, "bsw_direct_tables: support must lie in [2, 4096]");
    const int64_t n = L * S;
    k_direct_tables<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(endp, ers, mu, sc, ms, L, S, P, C);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

// ---- C ABI ---------------------------------------------------------------------------------------------------------------
extern "C" int bsw_direct_tables(const double *endp, int64_t ers, const double *mu, const double *sc, int64_t ms, int64_t L,
                                 int S, int bits, int quantbits, uint32_t *P, uint32_t *C, void *stream) {
    BSW_REQUIRE(bits == 31 && quantbits >= 0 && quantbits < bits, "bsw_direct_tables: bits must be 31, quantbits in [0, 31)");
    return bsw_direct_tables_st(endp, ers, mu, sc, ms, L, S, P, C, (cudaStream_t)stream);
}
static int abi_direct(bool pop, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc, int64_t sss,
                      const double *endp, int64_t ers, int16_t *sym, int64_t L, int S, int bits, int q, void *scratch,
                      int64_t scratch_bytes, cudaStream_t st) {
    if (int rc = direct_args_ok(s, first, count, mu, sc, endp, ers, sym, L, S, bits, q, scratch)) return rc;
    BSW_REQUIRE(scratch_bytes >= bsw_logistic_scratch_bytes(count, L, S, 0), "direct coder: scratch too small");
    if (int rc = bsw_direct_2p(0, pop, s, first, count, mu, mss, sc, sss, endp, ers, sym, L, S, scratch, scratch_bytes, nullptr, st)) return rc;
    return bsw_direct_2p(1, pop, s, first, count, mu, mss, sc, sss, endp, ers, sym, L, S, scratch, scratch_bytes, nullptr, st);
}
extern "C" int bsw_direct_push(bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc, int64_t sss,
                               const double *endp, int64_t ers, const int16_t *sym, int64_t L, int S, int bits, int q,
                               void *scratch, int64_t scratch_bytes, void *stream) {
    return abi_direct(false, s, first, count, mu, mss, sc, sss, endp, ers, (int16_t *)sym, L, S, bits, q, scratch, scratch_bytes,
                      (cudaStream_t)stream);
}
extern "C" int bsw_direct_pop(bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc, int64_t sss,
                              const double *endp, int64_t ers, int16_t *sym, int64_t L, int S, int bits, int q,
                              void *scratch, int64_t scratch_bytes, void *stream) {
    return abi_direct(true, s, first, count, mu, mss, sc, sss, endp, ers, sym, L, S, bits, q, scratch, scratch_bytes,
                      (cudaStream_t)stream);
}
