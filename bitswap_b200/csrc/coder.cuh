// Internal declarations of the ANS coder (ans_kernels.cu, ans_rows.cu, ans_rows6.cu; codec.cu calls in): the warp-level
// stream state, the two-phase scratch layout, the support dispatcher and the entry points shared between files.
#pragma once
#include <type_traits>
#include "bsw_common.cuh"

#define FULL 0xffffffffu

// Per-warp view of one stream with a 32-word register window over the top of the stack, so that the
// renormalisation words move to/from HBM as whole 128-byte lines.
struct WarpStream {
    uint32_t *words;   // this stream's row
    uint64_t x;        // head (replicated in all lanes)
    int len, cap;
    int wbase;         // index of the word lane 0 holds (multiple of 32), or -1
    uint32_t wbuf;     // lane j holds words[wbase + j]
    int err;

    __device__ __forceinline__ void open(const bsw_streams &sv, int b) {
        words = sv.words + (int64_t)b * sv.cap;
        x = sv.heads[b];
        len = sv.nwords[b];
        cap = (int)sv.cap;
        err = sv.flags[b];
        wbase = -1;
        wbuf = 0;
    }
    __device__ __forceinline__ void close(const bsw_streams &sv, int b, int lane) {
        if (lane == 0) { sv.heads[b] = x; sv.nwords[b] = len; sv.flags[b] = err; if (len < sv.minwords[b]) sv.minwords[b] = len; }
    }
    // ---- pop side: window slides downward -------------------------------------------------------
    __device__ __forceinline__ uint32_t pop_word(int lane) {     // caller guarantees len > 0
        int idx = len - 1;
        if (wbase < 0 || idx < wbase) {
            wbase = idx & ~31;
            wbuf = words[wbase + lane];
        }
        len = idx;
        return __shfl_sync(FULL, wbuf, idx - wbase);
    }
    // ---- push side: window slides upward --------------------------------------------------------
    __device__ __forceinline__ void push_begin(int lane) {
        wbase = len & ~31;
        wbuf = (wbase + lane < len) ? words[wbase + lane] : 0u;
    }
    __device__ __forceinline__ void push_word(uint32_t w, int lane) {   // caller guarantees len < cap
        if (lane == len - wbase) wbuf = w;
        ++len;
        if (len - wbase == 32) {
            words[wbase + lane] = wbuf;
            wbase += 32;
        }
    }
    __device__ __forceinline__ void push_end(int lane) {
        if (lane < len - wbase) words[wbase + lane] = wbuf;
    }
    // ---- the integer recurrences (cifar_compress.py:51-54 and :60-65) -------------------------------
    __device__ __forceinline__ void encode(uint32_t p, uint32_t c, int bits, int lane) {
        uint64_t lim = ((((uint64_t)1 << 32) >> bits) << 32) * (uint64_t)p;
        if (x >= lim) {
            if (len >= cap) { err = BSW_E_OVERFLOW; return; }
            push_word((uint32_t)x, lane);
            x >>= 32;
        }
        uint64_t qd = x / p;
        uint64_t rm = x - qd * p;
        x = (qd << bits) + rm + c;
    }
    // same recurrence with the division replaced by a multiply with M = floor((2^64-1)/p) computed in the parallel phase:
    // floor(x*M / 2^64) is floor(x/p) or one less, so a single correction makes it exact
    __device__ __forceinline__ void encode_magic(uint32_t p, uint32_t c, uint64_t M, int bits, int lane) {
        uint64_t lim = ((((uint64_t)1 << 32) >> bits) << 32) * (uint64_t)p;
        if (x >= lim) {
            if (len >= cap) { err = BSW_E_OVERFLOW; return; }
            push_word((uint32_t)x, lane);
            x >>= 32;
        }
        uint64_t qd = __umul64hi(x, M);
        uint64_t rm = x - qd * p;
        if (rm >= p) { rm -= p; ++qd; }
        x = (qd << bits) + rm + c;
    }
    __device__ __forceinline__ void decode(uint32_t p, uint32_t c, uint32_t m, int bits, int lane) {
        x = (uint64_t)p * (x >> bits) + m - c;
        if (x < ((uint64_t)1 << 32)) {
            if (len <= 0) { err = BSW_E_UNDERFLOW; return; }
            uint32_t w = pop_word(lane);
            x = (x << 32) | w;
        }
    }
};

__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v, int lane) {
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
__device__ __forceinline__ double shfl_d(double v, int src) {
    return __hiloint2double(__shfl_sync(FULL, __double2hiint(v), src), __shfl_sync(FULL, __double2loint(v), src));
}

// Scratch of the two-phase coder for `count` streams of L rows, for every support and both kernel families.  Push: one
// (P_s, C_s, reciprocal) uint4 per row.  Pop: the integer cdf at the start of each of the row's chunks (up to 32 u32 per
// row), then one (argmax, remnant) fix word per row.
struct RowsScratch {
    static constexpr size_t PUSH_ROW = 16, BASES_ROW = 32 * 4, POP_ROW = BASES_ROW + 8;
    uint4 *pairs;
    uint32_t *bases;
    uint2 *fix;
    RowsScratch(void *p, int count, int64_t L)
        : pairs((uint4 *)p), bases((uint32_t *)p), fix((uint2 *)((uint8_t *)p + (size_t)count * L * BASES_ROW)) {}
    static size_t bytes(bool pop, int count, int64_t L) { return (size_t)count * L * (pop ? POP_ROW : PUSH_ROW); }
};

// Calls f(std::integral_constant<int, S / 32>{}) for a support S in {32 * NB : NB = NB_LO, 2 NB_LO, ..., NB_HI}; any other
// S sets `msg` (with S appended) as the error and returns BSW_E_INVALID.
template <int NB_LO, int NB_HI, class F>
int with_support(int S, const char *msg, F &&f) {
    if (S == 32 * NB_LO) return f(std::integral_constant<int, NB_LO>{});
    if constexpr (NB_LO < NB_HI) return with_support<2 * NB_LO, NB_HI>(S, msg, f);
    bsw_set_error("%s (got %d)", msg, S);
    return BSW_E_INVALID;
}

// ---- entry points shared between the coder files and the codec ---------------------------------------------------------
// ans_kernels.cu: int16-symbol variants of the table-driven coder, the fused coder with block extents, rest-word marks
int bsw_ans_push_i16(bsw_streams *s, int first, int count, const uint32_t *P, const uint32_t *C, int64_t pss, int64_t css,
                     const int16_t *sym, int64_t L, int S, int bits, cudaStream_t st);
int bsw_ans_pop_i16(bsw_streams *s, int first, int count, const uint32_t *P, const uint32_t *C, int64_t pss, int64_t css,
                    int16_t *sym, int64_t L, int S, int bits, cudaStream_t st);
int bsw_logistic_fused_ext(bool push, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc,
                           int64_t sss, const double *endp, int64_t ers, int16_t *sym, int64_t L, int S, int bits, int q,
                           const int16_t *ext, cudaStream_t st);
int bsw_streams_mark_rest(bsw_streams *s, int first, int count, cudaStream_t st);
// ans_rows.cu: the two-phase coder and the shared-table prior pop
size_t bsw_rows_scratch_bytes(int count, int64_t L);
int bsw_rows_mode();
int bsw_prior_coarse(const uint32_t *C, int64_t L, int S, uint32_t *coarse, uint2 *fix, cudaStream_t st);
int bsw_pop_shared_table(bsw_streams *s, int first, int count, const uint32_t *P, const uint32_t *coarse, const uint2 *fix,
                         int16_t *sym, int64_t L, int S, int bits, cudaStream_t st);
int bsw_logistic_2p(int phase, bool pop, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc,
                    int64_t sss, const double *endp, int64_t ers, const void *meta, int16_t *sym, int64_t L, int S, int bits, int q,
                    void *scratch, size_t scratch_bytes, const int16_t *ext, cudaStream_t st);
int bsw_push_pairs(bsw_streams *s, int first, int count, const void *pairs, int64_t L, int bits, const int16_t *ext,
                   cudaStream_t st);
// ans_direct.cu: the direct-cdf coder
int bsw_direct_2p(int phase, bool pop, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc,
                  int64_t sss, const double *endp, int64_t ers, int16_t *sym, int64_t L, int S, void *scratch,
                  size_t scratch_bytes, const int16_t *ext, cudaStream_t st);
int bsw_direct_tables_st(const double *endp, int64_t ers, const double *mu, const double *sc, int64_t ms, int64_t L, int S,
                         uint32_t *P, uint32_t *C, cudaStream_t st);
// ans_rows6.cu: the affine-row kernels
int bsw_rows6_build_meta(const double *endp, int64_t ers, int64_t L, int S, void *meta_dev, int *n_affine_host, cudaStream_t st);
int bsw_rows6_launch(int phase, bool pop, bsw_streams *s, int first, int count, const float *mu, int64_t mss, const float *sc,
                     int64_t sss, const double *endp, int64_t ers, const void *meta, int16_t *sym, int64_t L, int S, int bits,
                     int q, void *scratch, size_t scratch_bytes, const int16_t *ext, cudaStream_t st);
