// Body of the tile kernels k_conv_wg<Args> (split arithmetic) and k_conv_bf16<Bf16<Args>> (single-pass bf16), included
// once into each (conv_tc.cu).  In scope: the tensor maps amap_hi, amap_lo, wmap_hi, wmap_lo, the tile arguments `a` of
// type Args and ntiles.  One text for both, and no wrapping function: the split kernels compile to exactly the code they
// had before the bf16 kernels existed.
    constexpr int N = Args::kN;
    using C = TileCfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    float *hand = (float *)(smem + C::NSTAGE * C::STAGE);
    uint64_t *full_bar = (uint64_t *)(smem + C::NSTAGE * C::STAGE + C::HAND);
    uint64_t *empty_bar = full_bar + C::NSTAGE;
    uint64_t *acc_full = empty_bar + C::NSTAGE, *acc_empty = acc_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = a.taps * a.cchunks;
    const bool mc = Args::kCoBlocks == 2 && cluster_nctarank() == 4;
    const uint32_t rank = mc ? cluster_ctarank() : 0;

    if (warp == PRODUCER_WARP && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&amap_hi) : "memory");
        if constexpr (!Args::kBf16) asm volatile("prefetch.tensormap [%0];" ::"l"(&amap_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap_hi) : "memory");
        if constexpr (!Args::kBf16) asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap_lo) : "memory");
        // empty: both consumer warpgroups of this CTA and, with multicast, of the peers this CTA writes into (two in the
        // split arithmetic, one in bf16)
        for (int s = 0; s < C::NSTAGE; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], mc ? (Args::kBf16 ? 4 : 6) : 2); }
        mbar_init(acc_full, 256);
        mbar_init(acc_empty, EPI_WARPS * 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // peers arrive on these barriers and multicast into this CTA's stages: all barriers of the cluster are initialised first
    if (mc) cluster_sync();
    else __syncthreads();

    if (warp >= PRODUCER_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS_EPILOGUE));
        if (warp >= EPI_WARP0) {     // ===== epilogue warps =====
            int it = 0;
            for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
                const int img = t / (2 * Args::kCoBlocks), co0 = ((t >> 1) % Args::kCoBlocks) * N, mh = t & 1;
                mbar_wait(acc_full, it & 1);
                epilogue<Args::kBf16>(a, hand, img, mh, co0, warp - EPI_WARP0, lane);
                mbar_arrive(acc_empty);
            }
        } else if (lane == 0) {     // ===== TMA producer =====
            const int r = a.ks / 2;
            const uint16_t amask = (uint16_t)(0x5u << (rank & 1)), wmask = (uint16_t)(0x3u << (rank & 2));
            int stage = 0, phase = 0;
            for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
                const int img = t / (2 * Args::kCoBlocks), co0 = ((t >> 1) % Args::kCoBlocks) * N, mh = t & 1;
                for (int kb = 0; kb < nkb; ++kb) {
                    const int tap = kb / a.cchunks, c0 = (kb - tap * a.cchunks) * BK;
                    const int dy = tap / a.ks, dx = tap - dy * a.ks;
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t *st = smem + stage * C::STAGE;
                    // whole stage (bf16: its hi boxes): the peers' boxes complete here too
                    mbar_expect_tx(&full_bar[stage], Args::kBf16 ? A_BYTES + C::W_BYTES : C::STAGE);
                    if constexpr (Args::kBf16) {
                        // A_hi of this pixel half by the CTA of channel block (rank & 1), W_hi of this channel block by the
                        // CTA of pixel half 1 - (rank >> 1): ranks 0 / 3 issue A, ranks 1 / 2 issue W
                        if (mc && (rank & 1) == (rank >> 1))
                            tma_load_4d_mc(st, &amap_hi, &full_bar[stage], amask, c0, dx - r, dy - r + 8 * mh, img);
                        else if (mc)
                            tma_load_3d_mc(st + 2 * A_BYTES, &wmap_hi, &full_bar[stage], wmask, c0, co0, tap);
                        else {
                            tma_load_4d(st, &amap_hi, &full_bar[stage], c0, dx - r, dy - r + 8 * mh, img);
                            tma_load_3d(st + 2 * A_BYTES, &wmap_hi, &full_bar[stage], c0, co0, tap);
                        }
                    } else if (mc) {
                        // A_hi by channel block 0, A_lo by block 1 of this pixel half; W_hi by pixel half 0, W_lo by half 1
                        const int ao = (rank & 2) ? A_BYTES : 0, wo = (rank & 1) ? C::W_BYTES : 0;
                        tma_load_4d_mc(st + ao, (rank & 2) ? &amap_lo : &amap_hi, &full_bar[stage], amask, c0, dx - r,
                                       dy - r + 8 * mh, img);
                        tma_load_3d_mc(st + 2 * A_BYTES + wo, (rank & 1) ? &wmap_lo : &wmap_hi, &full_bar[stage], wmask, c0,
                                       co0, tap);
                    } else {
                        tma_load_4d(st, &amap_hi, &full_bar[stage], c0, dx - r, dy - r + 8 * mh, img);
                        tma_load_4d(st + A_BYTES, &amap_lo, &full_bar[stage], c0, dx - r, dy - r + 8 * mh, img);
                        tma_load_3d(st + 2 * A_BYTES, &wmap_hi, &full_bar[stage], c0, co0, tap);
                        tma_load_3d(st + 2 * A_BYTES + C::W_BYTES, &wmap_lo, &full_bar[stage], c0, co0, tap);
                    }
                    if (++stage == C::NSTAGE) { stage = 0; phase ^= 1; }
                }
            }
            // Drain: wait for the last release of every stage.  With multicast, peers arrive on this CTA's barriers
            // until then, so the CTA must not exit before (a stage never filled passes at once: parity phase ^ 1).
            for (int s = 0; s < C::NSTAGE; ++s) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                if (++stage == C::NSTAGE) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS_CONSUMER));
    const int wg = warp >> 2;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);          // this thread's first accumulator row
    // one thread per warpgroup releases a stage: to this CTA's producer and, with multicast, to the peers writing into it
    // (bf16: the one other issuer of its two boxes, see the producer)
    auto release = [&](int s) {
        if ((threadIdx.x & 127) != 0) return;
        if constexpr (Args::kBf16) {
            if (mc) { mbar_arrive_cluster(&empty_bar[s], rank); mbar_arrive_cluster(&empty_bar[s], rank ^ ((rank & 1) == (rank >> 1) ? 1 : 2)); }
            else mbar_arrive(&empty_bar[s]);
        } else if (mc) { mbar_arrive_cluster(&empty_bar[s], rank); mbar_arrive_cluster(&empty_bar[s], rank ^ 1); mbar_arrive_cluster(&empty_bar[s], rank ^ 2); }
        else mbar_arrive(&empty_bar[s]);
    };
    // Folding tiles (Args::kFold): after the last k-block of every tap but the last, the consumers retire the MMAs in
    // flight, add the main accumulator into `outer` (float32 RNE adds) and restart it from zero, so the tensor core's
    // truncating accumulate never sums more than one tap's Wp terms into it.  In-convs (one k-block per tap) do not fold.
    constexpr bool fold = Args::kFold;
    const bool fold_taps = fold && a.cchunks > 1;
    int stage = 0, phase = 0, it = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
        float dm[N / 2], dc[N / 2], outer[fold ? N / 2 : 1];       // bf16: dc is never read
#pragma unroll
        for (int i = 0; i < N / 2; ++i) { dm[i] = 0.f; dc[i] = 0.f; }
        if constexpr (fold) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) outer[i] = 0.f;
        }
        int prev = -1, kc = 0;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sbase = smem_u32(smem + stage * C::STAGE);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {
                const uint64_t a_hi = make_desc_sw64(sbase + wg * (64 * BK * 2) + kk * 32);
                const uint64_t a_lo = make_desc_sw64(sbase + A_BYTES + wg * (64 * BK * 2) + kk * 32);
                const uint64_t b_hi = make_desc_sw64(sbase + 2 * A_BYTES + kk * 32);
                const uint64_t b_lo = make_desc_sw64(sbase + 2 * A_BYTES + C::W_BYTES + kk * 32);
                Wgmma<N>::mma(dm, a_hi, b_hi);
                if constexpr (!Args::kBf16) {                    // bf16: hi*hi only
                    Wgmma<N>::mma(dc, a_lo, b_hi);
                    Wgmma<N>::mma(dc, a_hi, b_lo);
                }
            }
            wg_commit();
            if (fold_taps && ++kc == a.cchunks && kb + 1 < nkb) {
                kc = 0;
                wg_wait<0>();                              // this tap's MMAs are done: both stages can go
                fence_regs(dm);
#pragma unroll
                for (int i = 0; i < N / 2; ++i) { outer[i] += dm[i]; dm[i] = 0.f; }
                if (prev >= 0) release(prev);
                release(stage);
                prev = -1;
            } else {
                wg_wait<1>();                              // the previous k-block's MMAs have read their stage
                if (prev >= 0) release(prev);
                prev = stage;
            }
            if (++stage == C::NSTAGE) { stage = 0; phase ^= 1; }
        }
        wg_wait<0>();
        fence_regs(dm);
        if constexpr (!Args::kBf16) fence_regs(dc);
        if (prev >= 0) release(prev);
        mbar_wait(acc_empty, (it & 1) ^ 1);            // the epilogue has read the previous tile
        hand_store<Args::kBf16>(a, hand, outer, dm, dc, row0, lane);
        mbar_arrive(acc_full);
    }
