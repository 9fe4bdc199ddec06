// Images in and out of the codec's block buffers on the device (include/bitswap_b200.h, bsw_tile_blocks /
// bsw_untile_regions): byte copies between strided HWC images and the [step, stream, C, 32, 32] buffers the encoder reads
// and the decoder writes.  The tables are sized by images + chains + regions, never by blocks: every thread finds its
// chain, image or region by binary search over prefix offsets, so a 2^24-block archive needs no per-block table.
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "bsw_common.cuh"

namespace {
constexpr int TL_THREADS = 256;
constexpr int64_t TL_MAX_BLOCKS = BSW_MAX_IMAGE_BLOCKS;

// last k in [0, n) with a[k] <= v, for a non-decreasing a with a[0] <= v
__host__ __device__ __forceinline__ int tl_find(const int64_t *a, int n, int64_t v) {
    int lo = 0, hi = n;                                              // a[lo] <= v < a[hi] (a[n] = +inf)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// Block grid of an h x w image: crop (and hwc_quirk) floors, code ceils.
__host__ __device__ __forceinline__ int64_t tl_grid(int64_t n, int mode) { return mode == BSW_TILE_CODE ? (n + 31) / 32 : n / 32; }

// One CTA per coded block q (stream order: stream j's blocks are cum[j] .. cum[j + 1]).  tab: ioff [n + 1] (first block of
// image i in the sequence), img [n][6] (base, sy, sx, sc, h, w), cum [K + 1], sstart [K] (first sequence block of stream j).
// Each thread assembles four consecutive bytes of the slot and stores them as one word.
__global__ void __launch_bounds__(TL_THREADS) k_tile_blocks(const int64_t *__restrict__ tab, int n, int K, int C, int mode,
                                                            uint8_t *__restrict__ out, int16_t *__restrict__ ext) {
    const int64_t *ioff = tab, *img = ioff + n + 1, *cum = img + 6 * n, *sstart = cum + K + 1;
    const int64_t q = blockIdx.x;
    const int j = tl_find(cum, K, q);
    const int64_t t = q - cum[j], g = sstart[j] + t;
    const int i = tl_find(ioff, n, g);
    const int64_t *d = img + 6 * i;
    const uint8_t *p = reinterpret_cast<const uint8_t *>(d[0]);
    const int64_t sy = d[1], sx = d[2], sc = d[3], h = d[4], w = d[5];
    const int64_t b = g - ioff[i], gw = tl_grid(w, mode), by = b / gw, bx = b - by * gw;
    const int vh = (int)min((int64_t)32, h - 32 * by), vw = (int)min((int64_t)32, w - 32 * bx);
    const int64_t row = t * K + j;
    if (ext != nullptr && threadIdx.x == 0) {
        ext[2 * row] = (int16_t)vh;
        ext[2 * row + 1] = (int16_t)vw;
    }
    const uint8_t *org = p + 32 * by * sy + 32 * bx * sx;
    uint32_t *slot = reinterpret_cast<uint32_t *>(out + row * C * 1024);
    for (int e4 = threadIdx.x; e4 < C * 256; e4 += TL_THREADS) {
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int e = 4 * e4 + k;
            int c, pix;
            if (mode == BSW_TILE_QUIRK) { pix = e / C; c = e - pix * C; }      // the HWC block's bytes, flat
            else { c = e >> 10; pix = e & 1023; }                              // CHW
            const int r = min(pix >> 5, vh - 1), col = min(pix & 31, vw - 1);   // edge replication outside the extent
            v |= (uint32_t)__ldg(org + r * sy + col * sx + c * sc) << (8 * k);
        }
        slot[e4] = v;
    }
}

// Grid-stride over the pixels of every region (region r's pixels are roff[r] .. roff[r + 1], row-major, C bytes each).
// tab: roff [R + 1], reg [R][5] (i, y, x, h, w), ioff [n + 1], gw [n], cstart [K + 1], cstream [K].  Block g of chain c
// sits at step cstart[c + 1] - 1 - g of stream cstream[c].
__global__ void __launch_bounds__(TL_THREADS) k_untile_regions(const int64_t *__restrict__ tab, int R, int n, int K, int C,
                                                               int n_streams, int quirk, const uint8_t *__restrict__ blocks,
                                                               uint8_t *__restrict__ out) {
    const int64_t *roff = tab, *reg = roff + R + 1, *ioff = reg + 5 * R, *gws = ioff + n + 1, *cstart = gws + n,
                  *cstream = cstart + K + 1;
    const int64_t total = roff[R];
    for (int64_t p = (int64_t)blockIdx.x * TL_THREADS + threadIdx.x; p < total; p += (int64_t)gridDim.x * TL_THREADS) {
        const int r = tl_find(roff, R, p);
        const int64_t *rg = reg + 5 * r;
        const int64_t loc = p - roff[r], py = loc / rg[4], X = rg[2] + (loc - py * rg[4]), Y = rg[1] + py;
        const int i = (int)rg[0];
        const int64_t g = ioff[i] + (Y >> 5) * gws[i] + (X >> 5);
        const int c = tl_find(cstart, K, g);
        const int64_t row = (cstart[c + 1] - 1 - g) * n_streams + cstream[c];
        const uint8_t *slot = blocks + row * C * 1024;
        const int pix = (int)(Y & 31) * 32 + (int)(X & 31);
        for (int ch = 0; ch < C; ++ch) out[p * C + ch] = __ldg(slot + (quirk ? pix * C + ch : ch * 1024 + pix));
    }
}

// Uploads one int64 table, launches, frees: all on `st`, nothing synchronised.
template <typename F>
int tl_run(const std::vector<int64_t> &tab, cudaStream_t st, F launch) {
    int64_t *d = nullptr;
    BSW_CUDA(cudaMallocAsync(reinterpret_cast<void **>(&d), sizeof(int64_t) * tab.size(), st));
    cudaError_t e = cudaMemcpyAsync(d, tab.data(), sizeof(int64_t) * tab.size(), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        launch(d);
        e = cudaGetLastError();
    }
    cudaFreeAsync(d, st);
    BSW_CUDA(e);
    return BSW_OK;
}

// Checks the chain table shared by both calls: counts >= 0 summing to the sequence's blocks; cstart receives the prefix sums.
int tl_chains(const int64_t *nb, int K, int64_t total, std::vector<int64_t> &cstart) {
    cstart.assign(K + 1, 0);
    for (int c = 0; c < K; ++c) {
        BSW_REQUIRE(nb[c] >= 0 && nb[c] <= total, "chain with a negative block count or more blocks than the sequence");
        cstart[c + 1] = cstart[c] + nb[c];
        BSW_REQUIRE(cstart[c + 1] <= total, "the chains run past the end of the block sequence");
    }
    BSW_REQUIRE(cstart[K] == total, "the chains do not cover the block sequence");
    return BSW_OK;
}

// Image (h, w) -> its block count under `mode`, appended to ioff.
int tl_image(int64_t h, int64_t w, int mode, std::vector<int64_t> &ioff) {
    BSW_REQUIRE(h >= 1 && w >= 1, "image with no pixels");
    const int64_t nb = tl_grid(h, mode) * tl_grid(w, mode);
    BSW_REQUIRE(nb <= TL_MAX_BLOCKS, "image of more than BSW_MAX_IMAGE_BLOCKS blocks");
    ioff.push_back(ioff.back() + nb);
    return BSW_OK;
}
}  // namespace

extern "C" int bsw_tile_blocks(const bsw_image_view *images_host, int n_images, int channels, int mode,
                               const int64_t *chain_blocks_host, const int32_t *chain_stream_host, int n_chains,
                               int64_t steps, uint8_t *blocks_dev, int16_t *extents_dev, void *stream) {
    BSW_REQUIRE(images_host && chain_blocks_host && chain_stream_host && blocks_dev, "bsw_tile_blocks: null pointer");
    BSW_REQUIRE(n_images >= 1 && n_chains >= 1 && steps >= 1, "bsw_tile_blocks: need an image, a chain and a step");
    BSW_REQUIRE(channels >= 1 && channels <= 4, "bsw_tile_blocks: channels must be 1 to 4");
    BSW_REQUIRE(mode == BSW_TILE_CROP || mode == BSW_TILE_CODE || mode == BSW_TILE_QUIRK, "bsw_tile_blocks: unknown mode");
    std::vector<int64_t> ioff{0}, img;
    img.reserve(6 * (size_t)n_images);
    for (int i = 0; i < n_images; ++i) {
        const bsw_image_view &v = images_host[i];
        BSW_REQUIRE(v.pixels, "bsw_tile_blocks: image with a null pixel pointer");
        BSW_REQUIRE(v.sy >= 0 && v.sx >= 0 && v.sc >= 0, "bsw_tile_blocks: negative stride");
        if (int rc = tl_image(v.h, v.w, mode, ioff)) return rc;
        for (int64_t f : {(int64_t)(uintptr_t)v.pixels, v.sy, v.sx, v.sc, (int64_t)v.h, (int64_t)v.w}) img.push_back(f);
    }
    BSW_REQUIRE(ioff.back() <= INT32_MAX, "bsw_tile_blocks: more than 2^31 - 1 blocks");
    std::vector<int64_t> cstart;
    if (int rc = tl_chains(chain_blocks_host, n_chains, ioff.back(), cstart)) return rc;
    // stream order: stream j holds chain c with chain_stream[c] == j; a permutation of [0, n_chains)
    std::vector<int> chain_of(n_chains, -1);
    for (int c = 0; c < n_chains; ++c) {
        const int j = chain_stream_host[c];
        BSW_REQUIRE(j >= 0 && j < n_chains && chain_of[j] < 0, "bsw_tile_blocks: chain streams are not a permutation");
        BSW_REQUIRE(chain_blocks_host[c] <= steps, "bsw_tile_blocks: a chain has more blocks than there are steps");
        chain_of[j] = c;
    }
    std::vector<int64_t> tab = ioff;
    tab.insert(tab.end(), img.begin(), img.end());
    tab.push_back(0);
    for (int j = 0; j < n_chains; ++j) tab.push_back(tab.back() + chain_blocks_host[chain_of[j]]);
    for (int j = 0; j < n_chains; ++j) tab.push_back(cstart[chain_of[j]]);
    const int64_t total = ioff.back();
    if (total == 0) return BSW_OK;                                      // crop mode, every image under 32 x 32
    return tl_run(tab, (cudaStream_t)stream, [&](const int64_t *d) {
        k_tile_blocks<<<(unsigned)total, TL_THREADS, 0, (cudaStream_t)stream>>>(
            d, n_images, n_chains, channels, mode, blocks_dev, mode == BSW_TILE_CODE ? extents_dev : nullptr);
    });
}

extern "C" int bsw_untile_regions(const int32_t *shapes_host, int n_images, int channels, int mode,
                                  const int64_t *chain_blocks_host, const int32_t *chain_stream_host, int n_chains,
                                  int n_streams, int64_t steps, const uint8_t *blocks_dev, const int32_t *regions_host,
                                  int n_regions, uint8_t *out_dev, void *stream) {
    BSW_REQUIRE(shapes_host && chain_blocks_host && chain_stream_host && blocks_dev && regions_host && out_dev,
                "bsw_untile_regions: null pointer");
    BSW_REQUIRE(n_images >= 1 && n_chains >= 1 && n_streams >= 1 && steps >= 1 && n_regions >= 1,
                "bsw_untile_regions: need an image, a chain, a stream, a step and a region");
    BSW_REQUIRE(channels >= 1 && channels <= 4, "bsw_untile_regions: channels must be 1 to 4");
    BSW_REQUIRE(mode == BSW_TILE_CROP || mode == BSW_TILE_CODE || mode == BSW_TILE_QUIRK, "bsw_untile_regions: unknown mode");
    std::vector<int64_t> ioff{0}, gws;
    for (int i = 0; i < n_images; ++i) {
        if (int rc = tl_image(shapes_host[2 * i], shapes_host[2 * i + 1], mode, ioff)) return rc;
        gws.push_back(tl_grid(shapes_host[2 * i + 1], mode));
    }
    std::vector<int64_t> cstart;
    if (int rc = tl_chains(chain_blocks_host, n_chains, ioff.back(), cstart)) return rc;
    for (int c = 0; c < n_chains; ++c)
        BSW_REQUIRE(chain_stream_host[c] >= -1 && chain_stream_host[c] < n_streams, "bsw_untile_regions: chain stream out of range");
    std::vector<int64_t> roff{0}, reg;
    for (int r = 0; r < n_regions; ++r) {
        const int32_t *q = regions_host + 5 * r;
        const int64_t i = q[0], y = q[1], x = q[2], h = q[3], w = q[4];
        BSW_REQUIRE(i >= 0 && i < n_images, "bsw_untile_regions: region of no image");
        const int64_t H = shapes_host[2 * i], W = shapes_host[2 * i + 1];
        const int64_t Hc = mode == BSW_TILE_CODE ? H : H - H % 32, Wc = mode == BSW_TILE_CODE ? W : W - W % 32;
        BSW_REQUIRE(h >= 1 && w >= 1 && y >= 0 && x >= 0 && y + h <= Hc && x + w <= Wc,
                    "bsw_untile_regions: region empty or outside its image");
        // every chain holding a block of the region is decoded, down to the region's earliest block in it
        const int64_t gw = gws[i], by0 = y / 32, by1 = (y + h - 1) / 32, bx0 = x / 32, bx1 = (x + w - 1) / 32;
        const int64_t gmin = ioff[i] + by0 * gw + bx0, gmax = ioff[i] + by1 * gw + bx1;
        for (int c = tl_find(cstart.data(), n_chains, gmin); c < n_chains && cstart[c] <= gmax; ++c) {
            const int64_t e = std::max(cstart[c], gmin) - ioff[i];
            int64_t rr = e / gw, cc = e % gw;
            if (cc < bx0) cc = bx0;
            else if (cc > bx1) { ++rr; cc = bx0; }
            const int64_t g = ioff[i] + rr * gw + cc;
            if (rr > by1) break;
            if (g >= cstart[c + 1]) continue;
            BSW_REQUIRE(chain_stream_host[c] >= 0 && cstart[c + 1] - 1 - g < steps,
                        "bsw_untile_regions: a region needs a block its chain's stream was not decoded to");
        }
        roff.push_back(roff.back() + h * w);
        for (int64_t f : {i, y, x, h, w}) reg.push_back(f);
    }
    std::vector<int64_t> tab = roff;
    tab.insert(tab.end(), reg.begin(), reg.end());
    tab.insert(tab.end(), ioff.begin(), ioff.end());
    tab.insert(tab.end(), gws.begin(), gws.end());
    tab.insert(tab.end(), cstart.begin(), cstart.end());
    for (int c = 0; c < n_chains; ++c) tab.push_back(chain_stream_host[c]);
    const int64_t grid = std::min<int64_t>((roff.back() + TL_THREADS - 1) / TL_THREADS, 8192);
    return tl_run(tab, (cudaStream_t)stream, [&](const int64_t *d) {
        k_untile_regions<<<(unsigned)grid, TL_THREADS, 0, (cudaStream_t)stream>>>(
            d, n_regions, n_images, n_chains, channels, n_streams, mode == BSW_TILE_QUIRK, blocks_dev, out_dev);
    });
}
