/*
 * bitswap_b200.h -- C ABI of the H100-native Bit-Swap hot path.
 *
 * The reference (fhkingma/bitswap @ dfe0bf7d) is pure Python and has no FFI: its
 * "plugin interface" for this path is a handful of Python call signatures
 * (SURVEY.md 8b).  Each entry point below names the reference call it replaces.
 * Python binds these with ctypes (bitswap_b200/_lib.py); INTEGRATION.md shows the
 * stub a maintainer of the reference would add to cifar_compress.py.
 *
 * Conventions
 *   - every function returns a bsw_status (0 = ok); nothing throws across the ABI
 *   - "dev" pointers are CUDA device pointers owned by the caller (e.g. torch
 *     tensors); the library never frees them.  "host" pointers are ordinary memory.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); every
 *     kernel is enqueued on it, no call synchronises unless it says so.
 *   - an ANS stream == one reference state list: 32-bit words bottom-first plus a
 *     64-bit head (cifar_compress.py:157-159).  B streams = B independent chains.
 */
#ifndef BITSWAP_B200_H
#define BITSWAP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    BSW_OK          = 0,
    BSW_E_UNDERFLOW = 1,   /* reference: IndexError from x.pop(-2)          (cifar_compress.py:65)    */
    BSW_E_OVERFLOW  = 2,   /* word stack capacity exhausted (reference lists grow without bound)      */
    BSW_E_BADTABLE  = 3,   /* reference: AssertionError on the cdf table    (cifar_compress.py:45-46) */
    BSW_E_INVALID   = 4,   /* bad argument                                                            */
    BSW_E_CUDA      = 5    /* CUDA runtime error; see bsw_last_error()                                */
} bsw_status;

const char *bsw_last_error(void);
int         bsw_version(void);
/* 1 if this build contains the tensor-core (wgmma) conv path (bsw_model_desc.use_tensor_cores may be set). */
int         bsw_has_tensor_cores(void);
/* Measures this GPU's peak float64 FMA rate (DFMA/s, lanes) with a register-resident kernel: the roofline
 * denominator of the float64 row-table kernel (the driver's MEASURED_PEAKS.json has no FP64 figure). */
int         bsw_measure_fp64_peak(double *dfma_per_s);
/* Device self-test: the lean cdf of the throughput kernels vs the exact (IEEE division + libdevice exp) cdf on n
 * random finite (endpoint, mu, sigma) triples, far tails included.  example_host: 5 doubles or NULL. */
int         bsw_selftest_cdf(int64_t n, uint64_t seed, int64_t *mismatches_host, double *example_host);
/* worst |screening cdf - exact cdf| over n random arguments, in units of 2^-51 (the screening window is 64 units) */
int         bsw_selftest_cdf_apx(int64_t n, uint64_t seed, double *worst_units_host);
/* Test hook: runs ONE conv of a finalized model -- the one loaded under the state_dict prefix `prefix`; a head goes by
 * its mu prefix ("infer_mu", "deepgen_mu.0.0", "gen_mu.0") -- for images [0, n), through the same per-conv dispatch
 * as bsw_vae_*: tensor-core dense conv / in-conv / head, SIMT in-conv followed by the bf16 split, or SIMT head after a
 * tensor-core trunk.  The role comes from the model's net plans.
 *   in_dev:  flat CHW `given` [n, dim] for in-convs; float32 NHWC [n,256,Wp] for dense convs and heads (padded
 *            channels zero).  On the tensor-core path it is split into the input planes as bsw_vae_* splits the trunk.
 *   flags:   epilogue of in-convs and dense convs, r = conv + bias: BSW_CONV_RESID r += T_dev (the residual, updated in
 *            place), BSW_CONV_T writes T_dev = (T_ELU ? ELU(r) : r), BSW_CONV_A writes the next conv's input
 *            (A_ELU ? ELU(T) : T) to A_dev (SIMT; NULL = an internal buffer) or to bf16 hi/lo planes (tensor cores).
 *   T_dev, A_dev: float32 [n,256,Wp].  planes_dev: uint16 [2][max_batch,256,Wp] (hi, lo) receives the whole plane
 *            buffer the conv wrote, pre-filled with 0xffff; tensor-core path with BSW_CONV_A only.
 *   mu_dev, scale_dev: head outputs [n, dim_out] flat CHW, as bsw_vae_* returns them (scale only with a scale head). */
#define BSW_CONV_RESID 1
#define BSW_CONV_T     2
#define BSW_CONV_T_ELU 4
#define BSW_CONV_A     8
#define BSW_CONV_A_ELU 16
int         bsw_selftest_conv(struct bsw_model *m, const char *prefix, const float *in_dev, int64_t n, int flags,
                              float *T_dev, float *A_dev, uint16_t *planes_dev, float *mu_dev, float *scale_dev,
                              void *stream);

/* ------------------------------------------------------------------------------------------------
 * Stream sets: B device-resident ANS states.
 * Replaces: the Python list `state` (cifar_compress.py:157-159) -- create/import == building the
 * list, export == reading it back / pickle.dump (cifar_compress.py:265-266).
 * ---------------------------------------------------------------------------------------------- */
typedef struct bsw_streams bsw_streams;
typedef struct bsw_bins bsw_bins;

/* capacity_words is rounded up to a multiple of 32. */
int bsw_streams_create(bsw_streams **out, int n_streams, int64_t capacity_words);
int bsw_streams_destroy(bsw_streams *s);
int bsw_streams_count(const bsw_streams *s);
int64_t bsw_streams_capacity(const bsw_streams *s);

/* Host import: stream (first+i) receives words_host[offsets[i] .. offsets[i+1]) and heads_host[i].
 * Synchronous. */
int bsw_streams_import(bsw_streams *s, int first, int count, const uint32_t *words_host,
                       const int64_t *offsets_host, const uint64_t *heads_host);
/* Every stream receives the same words/head (the reference seeds every experiment identically,
 * cifar_compress.py:93,157).  Synchronous. */
int bsw_streams_fill(bsw_streams *s, const uint32_t *words_host, int64_t nwords, uint64_t head);
/* Word counts (list length - 1), heads and per-stream status flags (bsw_status values). Synchronous. */
int bsw_streams_sizes(bsw_streams *s, int64_t *nwords_host, uint64_t *heads_host, int32_t *flags_host);
/* Lowest word count each stream has reached since import/fill: the part of the initial random words that was never
 * borrowed and can be trimmed from a stored bitstream (demo_compress.py:137,160 `excess_state_len`). Synchronous. */
int bsw_streams_min_words(bsw_streams *s, int64_t *min_host);
/* The reference's len(restbits) - 1 for each stream's chain since import/fill/unpack (-1: not reached yet), from which it
 * reports `totalbits` and the cumulative moving average (cifar_compress.py:253-259): the word count after the first
 * image's first pop for Bit-Swap (:190-192), after all nz pops of the first image for BB-ANS (:224-226).  Recorded by
 * bsw_codec_encode.  Synchronous. */
int bsw_streams_rest_words(bsw_streams *s, int64_t *rest_host);
/* Packed export: stream i's words go to words_host[offsets_host[i] ...). Synchronous. */
int bsw_streams_export(bsw_streams *s, int first, int count, uint32_t *words_host, const int64_t *offsets_host);
/* Device-side packed (de)serialisation, async on `stream`: all streams' words gathered into one contiguous device
 * buffer (capacity >= total words; offsets_dev holds count+1 int64 prefix sums, heads_dev count uint64), or scattered back
 * (unpack resets flags and rest words like import; a stream whose packed length exceeds its capacity is flagged
 * BSW_E_OVERFLOW and left otherwise untouched).  A host export is then three memcpys. */
int bsw_streams_pack(bsw_streams *s, int first, int count, uint32_t *words_dev, int64_t *offsets_dev, uint64_t *heads_dev,
                     void *stream);
int bsw_streams_unpack(bsw_streams *s, int first, int count, const uint32_t *words_dev, const int64_t *offsets_dev,
                       const uint64_t *heads_dev, void *stream);
/* Trimmed forms: only words[base_b .. n_b) of every stream travel, base_b = the lowest depth the stack ever reached
 * (bsw_streams_min_words) -- the initial random words below it were never borrowed and the receiver re-creates them from
 * the seed (demo_compress.py:137,160; demo_decompress.py:176-186).  base_dev: int32 [count], written by pack, read by
 * unpack.  unpack_trimmed writes above base_b into streams that already hold the initial words (bsw_streams_fill /
 * import), and flags BSW_E_OVERFLOW instead of writing past a stream's capacity. */
int bsw_streams_pack_trimmed(bsw_streams *s, int first, int count, uint32_t *words_dev, int64_t *offsets_dev,
                             uint64_t *heads_dev, int32_t *base_dev, void *stream);
int bsw_streams_unpack_trimmed(bsw_streams *s, int first, int count, const uint32_t *words_dev, const int64_t *offsets_dev,
                               const uint64_t *heads_dev, const int32_t *base_dev, void *stream);
/* Raw device views for device-resident pipelines (NCCL gathers, custom kernels). */
int bsw_streams_device_ptrs(bsw_streams *s, uint32_t **words_dev, int32_t **nwords_dev, uint64_t **heads_dev,
                            int32_t **flags_dev);
/* Device-side: sum over streams of (nwords) -> *total_dev (int64), async on `stream`. */
int bsw_streams_total_words(bsw_streams *s, int64_t *total_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a1  ANS.__init__ (cifar_compress.py:13-46): float64 pmfs [L,S] -> integer tables.
 *     P_dev [L,S] uint32, C_dev [L,S+1] uint32 (C[:,S] == 2^bits).  err_dev (int32, may be NULL) is
 *     set to BSW_E_BADTABLE if a row fails the reference's assertions.
 * ---------------------------------------------------------------------------------------------- */
int bsw_ans_tables(const double *pmfs_dev, int64_t L, int S, int bits, int quantbits,
                   uint32_t *P_dev, uint32_t *C_dev, int32_t *err_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a2/a3  ANS.encode / ANS.decode (cifar_compress.py:48-67) over given integer tables, batched over
 *     the set's streams [first, first+count).  Tables: P [.,L,S], C [.,L,S+1]; table_stream_stride
 *     = elements between consecutive streams' tables (0: one table shared by all streams).
 *     Symbols: int32 [count, L].  push walks rows ascending, pop descending, exactly as the
 *     reference loops do.
 * ---------------------------------------------------------------------------------------------- */
int bsw_ans_push(bsw_streams *s, int first, int count, const uint32_t *P_dev, const uint32_t *C_dev,
                 int64_t P_stream_stride, int64_t C_stream_stride, const int32_t *sym_dev,
                 int64_t L, int S, int bits, void *stream);
int bsw_ans_pop(bsw_streams *s, int first, int count, const uint32_t *P_dev, const uint32_t *C_dev,
                int64_t P_stream_stride, int64_t C_stream_stride, int32_t *sym_dev,
                int64_t L, int S, int bits, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a4  logistic_cdf + pmf assembly (utils/torch/rand.py:67-68, cifar_compress.py:182-184).
 *     endpoints_dev: row r starts at endpoints_dev + r*endp_row_stride and holds S-1 doubles
 *     (stride 0 = one row shared by all, as ImageBins' identical rows allow).
 *     mu/scale: double, indexed [r*ms] (ms = 0 broadcasts, as the prior does at :245).
 *     Writes pmfs_dev [L,S] float64 -- the debug/export path of the parity ladder (P2); the hot
 *     path never materialises pmfs.
 * ---------------------------------------------------------------------------------------------- */
int bsw_logistic_pmfs(const double *endpoints_dev, int64_t endp_row_stride, const double *mu_dev,
                      const double *scale_dev, int64_t ms, int64_t L, int S, double *pmfs_dev, void *stream);

/* a4+a1 fused, materialised: integer tables straight from (endpoints, mu, scale).  Used for tables
 * that are shared by every stream (the Logistic(0,1) prior, cifar_compress.py:245-247). */
int bsw_logistic_tables(const double *endpoints_dev, int64_t endp_row_stride, const double *mu_dev,
                        const double *scale_dev, int64_t ms, int64_t L, int S, int bits, int quantbits,
                        uint32_t *P_dev, uint32_t *C_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a4+a1+a2 / a4+a1+a3 fused hot kernels: one warp per stream builds each row's table in registers
 * (float64 logistic cdf -> trunc -> remnant at the row argmax -> scan) and codes the symbol; tables
 * never reach HBM.  Replaces the per-level sequence
 *     cdfs = logistic_cdf(...); pmfs = ...; ANS(pmfs, bits, q).encode/decode(state, ...)
 * of cifar_compress.py:182-187,197-202.
 *     mu_dev/scale_dev: float32 (the nets' outputs, up-cast to float64 in the kernel as
 *     model/cifar_train.py:375-376 does); element [b*mu_stream_stride + r].  A stream stride of 0
 *     shares the vector between streams (the unconditional x-scale, cifar_train.py:411).
 *     endpoints as above but each row holds S doubles, the last one +inf (library layout, see
 *     bsw_bins_*).  S must be a multiple of 32 and <= 1024: the fused kernels keep a row's table in one warp's
 *     registers.  Wider supports (S = 2048, 4096: quantbits 11, 12) go through the two-phase entry points below.
 *     sym: int16 [count, L].
 * ---------------------------------------------------------------------------------------------- */
int bsw_logistic_push(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                      const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                      int64_t endp_row_stride, const int16_t *sym_dev, int64_t L, int S, int bits,
                      int quantbits, void *stream);
int bsw_logistic_pop(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                     const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                     int64_t endp_row_stride, int16_t *sym_dev, int64_t L, int S, int bits,
                     int quantbits, void *stream);

/* Two-phase variants (the throughput path of the codec): a fully parallel float64 row-table kernel followed by the
 * serial integer coder; same arguments and bit-identical results, plus caller-provided 16-byte aligned device scratch
 * of at least bsw_logistic_scratch_bytes(count, L, S, 0) bytes (the last argument is ignored; kept for ABI stability).
 * Two kernel families: the generic one (any sorted endpoint rows) and the affine-row one for rows that are uniform
 * grids -- which is every row discretize_kbins() builds (discretization.py:105-118) and the ImageBins pixel row
 * (utils/torch/rand.py:146-147).  These two entry points probe the rows on every call (one small kernel + a stream
 * synchronise); the codec uses the classification bsw_bins_create made.
 * S: a power of two from 32 to 4096 (quantbits up to 12) for the generic family; a multiple of 4 in [8, 1024], 2048 or
 * 4096 for the affine one.  The scratch size does not depend on S (136 bytes per row and stream for a pop). */
int64_t bsw_logistic_scratch_bytes(int count, int64_t L, int S, int full_tables);
/* Kernel family for bsw_logistic_*_2p and the codec: -1 = by row classification (default; BSW_ROWS_MODE overrides),
 * 0 = generic kernels only, 1 = affine-row kernels for every row (non-uniform rows take the exact path per bin). */
int bsw_set_rows_mode(int mode);
/* 1 if every endpoint row of `level` (or the pixel row, level = -1) is a uniform grid. */
int bsw_bins_level_is_uniform(const bsw_bins *b, int level);
/* Debug: with verify on, every affine-row table launch also evaluates the exact function for every bin.
 * bsw_rows6_verify_read returns and resets {bins that differ from the exact function (must be 0), worst error of a
 * trusted bin in thousandths of its window, bins checked, bins that took the exact path}. */
int bsw_rows6_set_verify(int on);
/* Mapping of the affine-row table kernel: lanes of a warp that share one row (2, 4, 8 or 32; 0 = default 4, i.e. eight
 * rows per warp).  Every setting emits the same integers; exposed for A/B timing and the parity test. */
int bsw_rows6_set_lanes_per_row(int lpr);
/* Launch shape of the tensor-core convolutions, a bit mask: 1 / 2 / 4 = dense 3x3 / dense 5x5 / in-convs and heads on a
 * persistent grid (one CTA per SM, or one four-CTA cluster per four SMs, walking half-image tiles); a clear bit = one
 * CTA per tile.  8 = dense convs and in-convs as single CTAs without TMA multicast (by default each image's four tiles
 * run as one cluster sharing their operand loads); no effect on a model of padded width other than 256, whose tiles
 * always run as single CTAs.  Bits 1 / 2 split the dense convs by kernel size: <= 3 (1x1, 3x3) / >= 5 (5x5, 7x7).
 * -1 = default (BSW_TC_PERSIST if set, else 7).  Bit-identical results. */
int bsw_set_conv_mode(int mode);
int bsw_rows6_verify_read(uint64_t *out4_host);
int bsw_logistic_push_2p(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                         const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                         int64_t endp_row_stride, const int16_t *sym_dev, int64_t L, int S, int bits, int quantbits,
                         void *scratch_dev, int64_t scratch_bytes, void *stream);
int bsw_logistic_pop_2p(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                        const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                        int64_t endp_row_stride, int16_t *sym_dev, int64_t L, int S, int bits, int quantbits,
                        void *scratch_dev, int64_t scratch_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * The direct-cdf coder: an opt-in quantiser with its OWN bitstreams (not the reference's).  Each bin's integer cdf
 * comes from that bin's float cdf alone, so no call needs a whole-row table:
 *     F_k = the float64 logistic cdf at endpoint k (== torch.sigmoid((e_k - mu) / sigma)), a NaN argument counting as 0
 *     C_0 = 0,  C_S = 2^31,  C_k = floor(RN(F_{k-1} * (2^31 - 2S))) + 2k  (k = 1 .. S-1),  P_k = C_{k+1} - C_k
 * Every P_k >= 1; the endpoint row's pad is never read.  The same formula codes latents, pixels (S = 256) and the prior.
 * bsw_direct_push / bsw_direct_pop take the arguments of bsw_logistic_*_2p (bits must be 31; quantbits does not enter the
 * quantiser) and the same scratch size.  The rows mode, the k_rows6 lanes-per-row and verify switches and the fused
 * coder do not apply to them.  bsw_direct_tables exports P [L,S] and C [L,S+1] as bsw_logistic_tables does (mu, scale
 * as double; the rows need only S-1 endpoints).
 * ---------------------------------------------------------------------------------------------- */
#define BSW_CODER_REFERENCE 0
#define BSW_CODER_DIRECT    1
int bsw_direct_push(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                    const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                    int64_t endp_row_stride, const int16_t *sym_dev, int64_t L, int S, int bits, int quantbits,
                    void *scratch_dev, int64_t scratch_bytes, void *stream);
int bsw_direct_pop(bsw_streams *s, int first, int count, const float *mu_dev, int64_t mu_stream_stride,
                   const float *scale_dev, int64_t scale_stream_stride, const double *endpoints_dev,
                   int64_t endp_row_stride, int16_t *sym_dev, int64_t L, int S, int bits, int quantbits,
                   void *scratch_dev, int64_t scratch_bytes, void *stream);
int bsw_direct_tables(const double *endpoints_dev, int64_t endp_row_stride, const double *mu_dev,
                      const double *scale_dev, int64_t ms, int64_t L, int S, int bits, int quantbits,
                      uint32_t *P_dev, uint32_t *C_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Bin tables on the device.
 * Replaces: the tensors returned by discretize() (discretization.py:9-99) and ImageBins
 * (utils/torch/rand.py:134-153); the library keeps its own padded copy (each endpoint row padded
 * with +1e300 to S entries so that cdf_{S-1} == 1 falls out of the same formula).
 * ---------------------------------------------------------------------------------------------- */
/* zendpoints_host [nz, zdim, S-1], zcentres_host [nz, zdim, S] float64 (reference layout); quantbits in [5, 12]
 * (S = 2^quantbits = 32 ... 4096; BSW_E_INVALID otherwise, before any allocation: the top level's kernels own S/32 bins
 * per lane).  Device memory: 16 * nz * zdim * S bytes (padded endpoints + centres), 1.07 GB for cifar8 at 12. */
int bsw_bins_create(bsw_bins **out, int nz, int zdim, int quantbits, int xdim,
                    const double *zendpoints_host, const double *zcentres_host);
int bsw_bins_destroy(bsw_bins *b);
/* Device views: padded z endpoints of a level [zdim, S]; z centres of a level [zdim, S]; the single
 * padded x endpoint row [256]. */
int bsw_bins_device_ptrs(bsw_bins *b, int level, const double **zend_dev, const double **zcen_dev,
                         const double **xend_dev);

/* a5  centre gathers (cifar_compress.py:180,195): symbols -> float32 values fed to the nets
 *     (float64 table value cast to float32, model/cifar_train.py:324,392).
 *     z: out[b,d] = (float) zcentres[level, d, sym[b,d]];  x: out[b,d] = (float)((x-127.5)/127.5). */
int bsw_gather_zcentres(const bsw_bins *b, int level, const int16_t *sym_dev, float *out_dev, int64_t n_streams,
                        void *stream);
int bsw_gather_xcentres(const uint8_t *x_dev, float *out_dev, int64_t n, void *stream);

/* ------------------------------------------------------------------------------------------------
 * f3  Sampling epilogue and bin fit of discretize() (discretization.py:30-118).
 * minmax_dev: uint32 [2 * dim] running extrema (order-preserving encoding), reset before a level.
 * bsw_discretize_sample: out[r,d] = float16(mu[r,d] + scale[r,d] * eps), eps = log(u) - log1p(-u) with u clamped to
 *   [bound, 1 - bound] (utils/torch/rand.py:6-20), and folds the float16 values into the extrema.  scale_row_stride 0 = one
 *   shared scale row.  bsw_discretize_fold: fold float16 samples produced elsewhere (the top-level prior draw).
 * bsw_discretize_edges: np.linspace(min, max, 2^q + 1) per dimension -> endpoints [dim][2^q - 1] and centres [dim][2^q]
 *   in float64 (KBinsDiscretizer strategy='uniform', discretization.py:105-118).
 * ---------------------------------------------------------------------------------------------- */
int bsw_discretize_reset(uint32_t *minmax_dev, int dim, void *stream);
int bsw_discretize_sample(const float *mu_dev, const float *scale_dev, int64_t scale_row_stride, const float *u_dev, float bound,
                          void *out_half_dev, uint32_t *minmax_dev, int64_t rows, int dim, void *stream);
int bsw_discretize_fold(const void *samples_half_dev, uint32_t *minmax_dev, int64_t rows, int dim, void *stream);
int bsw_discretize_edges(const uint32_t *minmax_dev, int dim, int quantbits, double *endpoints_dev, int64_t endp_row_stride,
                         double *centres_dev, int64_t cen_row_stride, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a8-a10  The inference-time VAE.
 * Replaces: Model.infer(i)(given) / Model.generate(i)(given) in compressing mode
 * (model/cifar_train.py:315-438; imagenetcrop_train.py:306-315,417) and the WnConv2d / ResNetLayer /
 * Squeeze2d / UnSqueeze2d forwards they run (utils/torch/modules.py:98-106,175-241).
 * ---------------------------------------------------------------------------------------------- */
typedef struct bsw_model bsw_model;
typedef struct {
    int32_t xc;            /* image channels C (xs = (C,32,32)) */
    int32_t nz;
    int32_t zchannels;
    int32_t nprocessing;
    int32_t kernel_size;   /* 1, 3, 5 or 7 (else BSW_E_INVALID): ResNet blocks of the levels, z in-convs, heads;
                              infer_in and the nprocessing blocks are always 5x5 */
    int32_t resdepth;
    int32_t reswidth;
    int32_t cond_xscale;   /* imagenetcrop: x-scale from a conv head */
    int32_t max_batch;     /* activations are preallocated for this many images */
    int32_t use_tensor_cores; /* 1: wgmma tensor-core path for the W->W convs (needs a padded width of 64, 128,
                                 ..., 512, i.e. reswidth 1..512); 0: fp32 SIMT (any width) */
} bsw_model_desc;

int bsw_model_create(bsw_model **out, const bsw_model_desc *desc);
int bsw_model_destroy(bsw_model *m);
/* Loads one WnConv2d by its reference state_dict prefix (e.g. "infer_res0.0.res252layer1.conv1"):
 * v [O,I,k,k], gain [O], b [O] float32 host arrays.  Weight normalisation
 * w = v * g/(||v||+1e-10), g = softplus(gain) if loggain else gain (modules.py:98-105) is folded here,
 * once.  Synchronous. */
int bsw_model_load_conv(bsw_model *m, const char *prefix, const float *v_host, const float *gain_host,
                        const float *b_host, int O, int I, int k, int loggain);
/* The unconditional x-scale parameter gen_std [C,32,32] (model/cifar_train.py:306-308). */
int bsw_model_load_gen_std(bsw_model *m, const float *gen_std_host);
/* Call after all tensors are loaded; checks completeness. */
int bsw_model_finalize(bsw_model *m);
/* Arithmetic of a tensor-core model's tensor-core convs, from the next net call on:
 *   BSW_TC_SPLIT (default): every operand split into bf16 hi + lo planes, three MMAs per multiply-add (hi*hi, lo*hi,
 *     hi*lo); mu/sigma within 1e-4 of the float32 reference model.
 *   BSW_TC_BF16: one MMA per multiply-add on the RNE-rounded bf16 operands (float32 accumulate, float32 trunk and
 *     residual stream); faster, mu/sigma a few 1e-3 off the reference.
 * The two give different mu/sigma, so a bitstream decodes only with a model in the arithmetic it was encoded in (as with
 * SIMT against tensor cores).  Convs a tensor-core model runs on the float32 SIMT kernel (in-convs with more than 32
 * input channels, heads with more than 32 outputs) stay float32 in both.  BSW_E_INVALID for any other value and for a
 * model created with use_tensor_cores = 0. */
#define BSW_TC_SPLIT 0
#define BSW_TC_BF16  1
int bsw_model_set_tc_precision(bsw_model *m, int precision);

/* given_dev float32 [n, dim_in] flat CHW (what `given.float()` is in the reference);
 * mu_dev/scale_dev float32 [n, dim_out] flat CHW.  For generate(0) without cond_xscale the scale does
 * not depend on the input: scale_dev receives the [xdim] vector replicated n times only if
 * scale_per_stream != 0, else one [xdim] row. */
int bsw_vae_infer(bsw_model *m, int level, const float *given_dev, int64_t n, float *mu_dev, float *scale_dev,
                  void *stream);
int bsw_vae_generate(bsw_model *m, int level, const float *given_dev, int64_t n, float *mu_dev, float *scale_dev,
                     int scale_per_stream, void *stream);

/* ------------------------------------------------------------------------------------------------
 * a11/a12  The Bit-Swap recursion, device resident.
 * Replaces: the sender loop body of cifar_compress.py:175-204,244-250 and the receiver loop body of
 * :283-317 for `count` streams at once (one image per stream per call; chain images by calling again).
 * x_dev uint8 [count, C,32,32].  No host round trip between levels; errors land in the per-stream
 * flags (bsw_streams_sizes).  `scheme`: 0 = Bit-Swap, 1 = BB-ANS (cifar_compress.py:205-242,319-352).
 * ---------------------------------------------------------------------------------------------- */
typedef struct bsw_codec bsw_codec;
int bsw_codec_create(bsw_codec **out, bsw_model *m, bsw_bins *b, int max_batch);
int bsw_codec_destroy(bsw_codec *c);
int bsw_codec_encode(bsw_codec *c, bsw_streams *s, int first, int count, const uint8_t *x_dev, int scheme,
                     void *stream);
int bsw_codec_decode(bsw_codec *c, bsw_streams *s, int first, int count, uint8_t *x_dev, int scheme,
                     void *stream);
/* The same calls for partial edge blocks of a larger image.  extent_dev int16 [count][2] on the device, indexed like x_dev:
 * the block's valid extent (vh, vw) in [1, 32]^2; NULL = full blocks (then identical to bsw_codec_encode/decode).
 * Only the pixel level changes: dims (c, r, col) with r >= vh or col >= vw are neither pushed nor popped (the order and
 * the tables of the coded dims are those of a full call), and before infer(0) both sides fill them by edge replication,
 * (c, min(r, vh-1), min(col, vw-1)) -- np.pad(mode="edge") of the valid region -- so the bitstream does not depend on
 * what the caller left there.  The decoder writes the padded blocks to x_dev.  A stream with an extent outside
 * [1, 32]^2 is flagged BSW_E_INVALID and left uncoded; the other streams are unaffected.  Needs xs = (C, 32, 32). */
int bsw_codec_encode_ext(bsw_codec *c, bsw_streams *s, int first, int count, const uint8_t *x_dev,
                         const int16_t *extent_dev, int scheme, void *stream);
int bsw_codec_decode_ext(bsw_codec *c, bsw_streams *s, int first, int count, uint8_t *x_dev,
                         const int16_t *extent_dev, int scheme, void *stream);
/* Number of kernel launches the last encode/decode call enqueued (bench.py's gpu_launches). */
int64_t bsw_codec_last_launches(const bsw_codec *c);
/* Stream placement inside one encode/decode call: 0 (default) = every kernel on the caller's stream; 1 = conv kernels
 * on a high-priority internal stream, coder kernels on a low-priority one, chained with events and joined back into
 * `stream` at the end (an experiment in co-scheduling tensor-bound and FP64-bound CTAs). */
int bsw_codec_set_dual_stream(bsw_codec *c, int on);
/* Coder variant: 1 (default) = two-phase (ans_rows.cu: fully parallel float64 row tables, then the serial integer
 * coder), 0 = fused one-warp-per-stream kernels (bsw_logistic_push/pop).  Bit-identical results.  0 is refused
 * (BSW_E_INVALID) when the codec's bins have more than 1024 bins per row (quantbits 11 and 12): the fused kernels
 * cannot hold such a table in registers, and on a codec set to the direct coder (the switch picks between reference
 * coders). */
int bsw_codec_set_two_phase(bsw_codec *c, int on);
/* Quantiser of every level and the prior, from the next encode or decode on: BSW_CODER_REFERENCE (default, the
 * reference's bitstreams) or BSW_CODER_DIRECT (see bsw_direct_push; its own bitstreams, decodable only by a direct codec).
 * The first switch to direct builds the direct prior tables and synchronises.  BSW_E_INVALID for any other value. */
int bsw_codec_set_coder(bsw_codec *c, int coder);
/* Per-kernel-category device time (CUDA events on the launching stream) accumulated since profiling was
 * enabled.  ms_out/n_out: 12 entries {misc, conv_in, conv_dense3x3, conv_dense5x5, conv_head, pop_z, push_z,
 * pop_x, push_x, prior, rows_z, rows_x} (rows_* = phase A of the two-phase coder; pop/push = phase B).  enable: 1 = reset and start, 0 = reset and stop, -1 = read only.  Synchronises. */
int bsw_codec_profile(bsw_codec *c, int enable, double *ms_out, int64_t *n_out);

/* ------------------------------------------------------------------------------------------------
 * Digests and the codec fingerprint (digest.cu): what a stored bitstream records about the codec that made it, so that a
 * decoder can refuse a bitstream it would decode into wrong pixels.  The digests catch accidental mismatches (another
 * checkpoint, other bins, a one-ulp difference in one weight); they are NOT cryptographic and do not resist tampering.
 *
 * bsw_digest: a 128-bit digest of `bytes` bytes at `dev` (device memory, 8-byte aligned), defined with integer operations
 * only, so it does not depend on the grid, the device or the batch:
 *   - the bytes are zero-padded to a multiple of 8 and read as little-endian uint64 words w[0 .. n);
 *   - chunk c holds words [8192 c, min(8192 (c + 1), n)); in it, lane l (0..31) starts from a = mix(64 c + 2 l),
 *     b = mix(64 c + 2 l + 1) and takes words 8192 c + l, + 32, + 64, ... in order:
 *         a = rotl(a ^ w, 29) * 0x9E3779B97F4A7C15,   b = (rotl(b, 23) + w) * 0xC2B2AE3D27D4EB4F;
 *   - the chunk's hash is ha = mix(c ^ 0x5354414D50484131), hb = mix(c + 0x5354414D50484232), then for l = 0 .. 31 in
 *     order ha = mix(ha ^ a_l), hb = mix(hb + b_l);
 *   - the digest starts from da = mix(bytes ^ 0x4449474553544131), db = mix(bytes + 0x4449474553544232) and folds the
 *     chunks in order: da = mix(da ^ ha_c), db = mix(db + hb_c);  out4 = {lo(da), hi(da), lo(db), hi(db)}.
 *   mix is the splitmix64 finaliser (z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB;
 *   z ^= z >> 31), arithmetic mod 2^64.  Every step is a bijection of the word it takes, so a change of one word always
 *   changes the digest.  Enqueued on `stream`; synchronises.
 * bsw_model_digest: the digest of the folded model the kernels read: the descriptor (xc, nz, zchannels, nprocessing,
 *   kernel_size, resdepth, reswidth, cond_xscale: not max_batch, not use_tensor_cores), then every conv slot in slot order
 *   (Cin, Cout, ks, CinP, CoutP, parts, the digests of its float32 weights w [taps][CinP][CoutP] and bias [CoutP]), then,
 *   without a conditional x-scale head, the digest of the folded x-scale [xdim].  The bf16 hi/lo planes are a function of
 *   w and are left out, as are activations.  Needs a finalized model; computed once and kept until a weight is reloaded.
 * bsw_bins_digest: the digest of (quantbits, nz, zdim) and of the padded z endpoints, the z centres and the x endpoints as
 *   stored on the device.  Computed once (bin tables are immutable).
 * ---------------------------------------------------------------------------------------------- */
/* Bump whenever a change alters mu/sigma or the integer tables under settings that exist already: bitstreams written by
 * an older revision then no longer match the codec, and stamped ones are refused instead of decoding into wrong pixels. */
#define BSW_BITSTREAM_REVISION 1
int bsw_bitstream_revision(void);
int bsw_digest(const void *dev, int64_t bytes, uint32_t out4[4], void *stream);
int bsw_model_digest(bsw_model *m, uint32_t out4[4], void *stream);
int bsw_bins_digest(bsw_bins *b, uint32_t out4[4], void *stream);

/* Everything that decides a codec's bitstreams.  Settings the parity tests show to be result-neutral are not in it: the
 * conv mode bits, the rows mode, the k_rows6 lanes per row and verify mode, two-phase vs fused reference coder, dual stream,
 * PipelinedCodec lanes and max_batch (see bsw_set_conv_mode, bsw_set_rows_mode, bsw_rows6_set_lanes_per_row,
 * bsw_codec_set_two_phase, bsw_codec_set_dual_stream). */
typedef struct {
    int32_t revision;                   /* BSW_BITSTREAM_REVISION of the library */
    int32_t xc, nz, zchannels, nprocessing, kernel_size, resdepth, reswidth, cond_xscale;   /* the model descriptor */
    int32_t quantbits;
    int32_t use_tensor_cores;           /* conv path: 1 = tensor cores, 0 = float32 SIMT */
    int32_t tc_precision;               /* BSW_TC_SPLIT / BSW_TC_BF16 (BSW_TC_SPLIT on a SIMT model) */
    int32_t tc_heads;                   /* 1 if any head runs on the tensor cores (0 with BSW_TC_HEADS=0) */
    int32_t coder;                      /* BSW_CODER_REFERENCE / BSW_CODER_DIRECT */
    uint32_t model_digest[4];           /* bsw_model_digest */
    uint32_t bins_digest[4];            /* bsw_bins_digest */
} bsw_fingerprint;
/* The codec as it is now (the coder it was last set to).  Synchronises the first time the digests are computed. */
int bsw_codec_fingerprint(bsw_codec *c, bsw_fingerprint *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Images in and out of the codec's block buffers (tiles.cu): byte copies on the device, so that images can enter and leave
 * as device memory and a host image crosses PCIe once, whole.
 *
 * A set of images is one block sequence: image i's blocks in row-major order over its block grid, the images in turn.  The
 * grid of an h x w image is floor(h/32) x floor(w/32) in BSW_TILE_CROP and BSW_TILE_QUIRK (the image cut down to multiples
 * of 32, every block full) and ceil(h/32) x ceil(w/32) in BSW_TILE_CODE (partial blocks at the bottom and right edges, valid
 * extent (vh, vw) = (min(32, h - 32 by), min(32, w - 32 bx)), as bsw_codec_encode_ext codes them).  A block is stored CHW,
 * [C][32][32]; BSW_TILE_QUIRK stores the block's HWC bytes [32][32][C] flat in the same C*1024 bytes instead.
 *
 * The sequence is cut into chains: chain_blocks_host[c] (int64 >= 0) blocks each, in sequence order, covering it exactly.
 * A block buffer is [steps][n_streams][C][32][32] uint8.  The tables are host memory, sized by images, chains and regions;
 * they are validated on the host before anything is uploaded or launched (BSW_E_INVALID, nothing enqueued), then copied
 * to the device in one transfer on `stream`.  The pixel memory behind a pointer cannot be checked: the caller guarantees
 * that every element the view addresses is readable device memory.
 * ---------------------------------------------------------------------------------------------- */
#define BSW_TILE_CROP  0
#define BSW_TILE_CODE  1
#define BSW_TILE_QUIRK 2
#define BSW_MAX_IMAGE_BLOCKS (1 << 20)   /* blocks per image either call accepts */
typedef struct {
    const uint8_t *pixels;   /* device: pixel (y, x) channel c is pixels[y * sy + x * sx + c * sc] */
    int32_t h, w;            /* >= 1 each, at most BSW_MAX_IMAGE_BLOCKS blocks */
    int64_t sy, sx, sc;      /* element strides, any value >= 0 (0 repeats a row, column or channel) */
} bsw_image_view;
/* The encoder's input: row (t, j) of blocks_dev (n_streams = n_chains) receives block t of the chain c with
 * chain_stream_host[c] == j (a permutation of [0, n_chains)), for t < chain_blocks_host[c] <= steps; rows past a chain's
 * end are not written.  Pixels outside a block's extent are edge-replicated.  BSW_TILE_CODE with extents_dev non-NULL
 * also writes int16 extents_dev[t][j] = (vh, vw) for the same rows.  1 <= channels <= 4; an image may have no blocks (crop
 * mode under 32 x 32), and if no image has any, nothing is enqueued. */
int bsw_tile_blocks(const bsw_image_view *images_host, int n_images, int channels, int mode,
                    const int64_t *chain_blocks_host, const int32_t *chain_stream_host, int n_chains, int64_t steps,
                    uint8_t *blocks_dev, int16_t *extents_dev, void *stream);
/* The decoder's output, cut: region r = regions_host[r] = (i, y, x, h, w) int32, inside image i (shapes_host[i] = (H, W),
 * cropped to multiples of 32 outside BSW_TILE_CODE), is written to out_dev as contiguous HWC uint8, the regions in
 * turn (region r starts at C times the pixels of the regions before it).  Block g of chain c (chain start s0, nb blocks)
 * is read from step s0 + nb - 1 - g of stream chain_stream_host[c] (-1: the chain was not decoded): the layout a decoder
 * that pops every chain from its end leaves.  Regions may share blocks and span blocks and chains; every block a region
 * needs must lie in a decoded chain at a step below `steps`. */
int bsw_untile_regions(const int32_t *shapes_host, int n_images, int channels, int mode,
                       const int64_t *chain_blocks_host, const int32_t *chain_stream_host, int n_chains, int n_streams,
                       int64_t steps, const uint8_t *blocks_dev, const int32_t *regions_host, int n_regions,
                       uint8_t *out_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Per-block pixel digests (checksums.cu): what a checked container or archive stores for every coded block, so that a
 * decoder can tell a block it decoded wrong from one it decoded right.  They catch accidents (another coder, arithmetic,
 * build or libm than the encoder's; a corrupt array), NOT tampering: nothing here is cryptographic.
 *
 * bsw_block_digest of one slot [C][32][32] of a block buffer (the layout of bsw_tile_blocks) that holds block i of its
 * block sequence (i counted from the sequence's first block) with valid extent (vh, vw) ((32, 32) for a full block and
 * for every BSW_TILE_QUIRK slot, whose C*1024 bytes are then covered in slot order), with integer operations only:
 *   - s = mix64(((i << 16) | (vh << 8) | vw) ^ 0x424C4F434B534551)                       (i < 2^31, vh, vw in [0, 32])
 *   - lane l = 0 .. 31 starts from a_l = lo32(mix64(s + l + 1)); if l < vw it takes the bytes x[c][r][l] for
 *     c = 0 .. C-1, and in each c r = 0 .. vh-1, in that order:   a_l = rotl32(a_l ^ x, 13) * 0x9E3779B1  (mod 2^32);
 *   - h = hi32(s), then for l = 0 .. 31 in order h = fmix32(h ^ a_l); the digest is h.
 *   mix64 is the splitmix64 finaliser of bsw_digest; fmix32 is murmur3's (h ^= h >> 16; h *= 0x85EBCA6B; h ^= h >> 13;
 *   h *= 0xC2B2AE35; h ^= h >> 16).  Every step is a bijection of the byte or word it takes, so one changed byte inside
 *   the extent always changes the digest; bytes outside it are not read.  The seed makes a block decoded into another
 *   place of the sequence, or with another extent, fail as well.
 *
 * A block buffer of n_slots slots (e.g. [steps][n_streams] flattened) and, per slot, block_host[q] (int64): the index of
 * the block it holds in one block sequence made of n_seqs sequences laid end to end, sequence k holding blocks
 * seq_offsets_host[k] .. seq_offsets_host[k + 1] (seq_offsets_host[0] = 0, non-decreasing, at most 2^31 - 1 in all), or
 * -1 for a slot to skip.  A block is digested as block g - seq_offsets_host[k] of its own sequence k.  extents_dev: int16
 * [n_slots][2] (vh, vw) on the device, or NULL for full blocks.  Validated on the host before anything is uploaded or
 * launched (BSW_E_INVALID, nothing enqueued): null pointers, n_slots, n_seqs >= 1, 1 <= channels <= 4, the offsets, every
 * block index in [-1, total) and no block in two slots.  Both calls are enqueued on `stream` and do not synchronise.
 * bsw_block_digests: digests_dev[g] (uint32 [total]) receives the digest of every block g in a slot; other entries are
 *   left alone.
 * bsw_block_digests_check: compares each such digest with expected_dev[g] (uint32 [total]) and writes result_dev (int64
 *   [2], device) = {blocks that differ, the lowest index g among them (INT64_MAX if none)}. */
int bsw_block_digests(const uint8_t *blocks_dev, const int16_t *extents_dev, int channels, int64_t n_slots,
                      const int64_t *block_host, const int64_t *seq_offsets_host, int n_seqs, uint32_t *digests_dev,
                      void *stream);
int bsw_block_digests_check(const uint8_t *blocks_dev, const int16_t *extents_dev, int channels, int64_t n_slots,
                            const int64_t *block_host, const int64_t *seq_offsets_host, int n_seqs,
                            const uint32_t *expected_dev, int64_t *result_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BITSWAP_B200_H */
