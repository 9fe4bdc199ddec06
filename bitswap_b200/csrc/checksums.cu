// Per-block pixel digests of the codec's block buffers (include/bitswap_b200.h, bsw_block_digests /
// bsw_block_digests_check): the writers store one 32-bit digest per coded block, and the decoders check every block they
// decode against it where the pixels already are, so that only a mismatch count and one block index come back to the host.
// Integer operations only, in a fixed order per lane and across lanes, so the result does not depend on the launch shape
// or the device.  Meant to catch accidental mismatches, not tampering: nothing here is cryptographic.
#include <stdint.h>
#include <vector>
#include "bsw_common.cuh"

namespace {
constexpr int BD_WARPS = 8;                                         // slots (warps) per CTA
constexpr uint64_t BD_SEED = 0x424C4F434B534551ull;                 // "BLOCKSEQ"
constexpr uint32_t BD_P = 0x9E3779B1u;
constexpr int64_t BD_MAX_BLOCKS = INT32_MAX;

__host__ __device__ __forceinline__ uint64_t bd_mix64(uint64_t z) {   // splitmix64 finaliser (a bijection)
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t bd_mix32(uint32_t h) {           // murmur3 fmix32 (a bijection)
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    return h ^ (h >> 16);
}
__device__ __forceinline__ uint32_t bd_step(uint32_t a, uint32_t x) { return __funnelshift_l(a ^ x, a ^ x, 13) * BD_P; }

// last k in [0, n) with a[k] <= v, for a non-decreasing a with a[0] <= v
__device__ __forceinline__ int bd_find(const int64_t *a, int n, int64_t v) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// One warp per slot q of blocks [n_slots][C][32][32]: lane l hashes column l of every channel's rows inside the extent,
// then the lane states are folded in lane order.  tab: block [n_slots] (sequence index, -1 = empty), off [n_seqs + 1].
// expected == nullptr: out[g] = the digest of block g.  Else the digest is compared with expected[g], and a mismatch
// counts in res[0] and lowers res[1] to g.
__global__ void __launch_bounds__(32 * BD_WARPS) k_block_digests(const uint8_t *__restrict__ blocks,
                                                                 const int16_t *__restrict__ ext, int C, int64_t n_slots,
                                                                 const int64_t *__restrict__ tab, int n_seqs,
                                                                 uint32_t *__restrict__ out,
                                                                 const uint32_t *__restrict__ expected,
                                                                 unsigned long long *__restrict__ res) {
    const int64_t q = (int64_t)blockIdx.x * BD_WARPS + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (q >= n_slots) return;                                               // warp-uniform
    const int64_t g = tab[q];
    if (g < 0) return;                                                      // an empty slot
    const int64_t *off = tab + n_slots;
    const int64_t i = g - off[bd_find(off, n_seqs, g)];
    int vh = 32, vw = 32;
    if (ext != nullptr) {                                                   // clamped: memory safety only, the codec
        vh = min(max((int)ext[2 * q], 0), 32);                              // never hands out such an extent
        vw = min(max((int)ext[2 * q + 1], 0), 32);
    }
    const uint64_t s = bd_mix64((((uint64_t)i << 16) | ((uint64_t)vh << 8) | (uint64_t)vw) ^ BD_SEED);
    uint32_t a = (uint32_t)bd_mix64(s + (uint64_t)lane + 1);
    if (lane < vw) {
        const uint8_t *slot = blocks + q * C * 1024 + lane;
        for (int c = 0; c < C; ++c) {
            const uint8_t *p = slot + c * 1024;
            int r = 0;
            for (; r + 8 <= vh; r += 8) {
                uint32_t v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = __ldg(p + (r + k) * 32);
#pragma unroll
                for (int k = 0; k < 8; ++k) a = bd_step(a, v[k]);
            }
            for (; r < vh; ++r) a = bd_step(a, __ldg(p + r * 32));
        }
    }
    uint32_t h = (uint32_t)(s >> 32);
    for (int l = 0; l < 32; ++l) h = bd_mix32(h ^ __shfl_sync(0xffffffffu, a, l));
    if (lane != 0) return;
    if (expected == nullptr) {
        out[g] = h;
    } else if (h != expected[g]) {
        atomicAdd(res, 1ull);
        atomicMin(reinterpret_cast<long long *>(res + 1), (long long)g);
    }
}

// Validates the shared arguments and builds the table: block [n_slots], then off [n_seqs + 1].  total: the blocks of the
// sequences, the length of the digest arrays.
int bd_table(const uint8_t *blocks_dev, int channels, int64_t n_slots, const int64_t *block_host,
             const int64_t *seq_offsets_host, int n_seqs, std::vector<int64_t> &tab, int64_t &total) {
    BSW_REQUIRE(blocks_dev && block_host && seq_offsets_host, "bsw_block_digests: null pointer");
    BSW_REQUIRE(n_slots >= 1 && n_seqs >= 1, "bsw_block_digests: need a slot and a sequence");
    BSW_REQUIRE(channels >= 1 && channels <= 4, "bsw_block_digests: channels must be 1 to 4");
    BSW_REQUIRE(n_slots <= (int64_t)BD_WARPS * INT32_MAX, "bsw_block_digests: too many slots");
    BSW_REQUIRE(seq_offsets_host[0] == 0, "bsw_block_digests: the first sequence must start at block 0");
    for (int s = 0; s < n_seqs; ++s)
        BSW_REQUIRE(seq_offsets_host[s + 1] >= seq_offsets_host[s] && seq_offsets_host[s + 1] <= BD_MAX_BLOCKS,
                    "bsw_block_digests: sequence offsets decrease or exceed 2^31 - 1 blocks");
    total = seq_offsets_host[n_seqs];
    std::vector<char> seen((size_t)total, 0);
    tab.assign(block_host, block_host + n_slots);
    for (int64_t q = 0; q < n_slots; ++q) {
        const int64_t g = block_host[q];
        BSW_REQUIRE(g >= -1 && g < total, "bsw_block_digests: block index out of range");
        if (g < 0) continue;
        BSW_REQUIRE(!seen[g], "bsw_block_digests: a block in two slots");
        seen[g] = 1;
    }
    tab.insert(tab.end(), seq_offsets_host, seq_offsets_host + n_seqs + 1);
    return BSW_OK;
}

// Uploads the table, launches, frees: all on `st`, nothing synchronised.
int bd_run(const std::vector<int64_t> &tab, const uint8_t *blocks, const int16_t *ext, int C, int64_t n_slots, int n_seqs,
           uint32_t *out, const uint32_t *expected, int64_t *res, cudaStream_t st) {
    int64_t *d = nullptr;
    BSW_CUDA(cudaMallocAsync(reinterpret_cast<void **>(&d), sizeof(int64_t) * tab.size(), st));
    cudaError_t e = cudaMemcpyAsync(d, tab.data(), sizeof(int64_t) * tab.size(), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && res != nullptr) {
        const int64_t init[2] = {0, INT64_MAX};
        e = cudaMemcpyAsync(res, init, sizeof(init), cudaMemcpyHostToDevice, st);
    }
    if (e == cudaSuccess) {
        k_block_digests<<<(unsigned)((n_slots + BD_WARPS - 1) / BD_WARPS), 32 * BD_WARPS, 0, st>>>(
            blocks, ext, C, n_slots, d, n_seqs, out, expected, reinterpret_cast<unsigned long long *>(res));
        e = cudaGetLastError();
    }
    cudaFreeAsync(d, st);
    BSW_CUDA(e);
    return BSW_OK;
}
}  // namespace

extern "C" int bsw_block_digests(const uint8_t *blocks_dev, const int16_t *extents_dev, int channels, int64_t n_slots,
                                 const int64_t *block_host, const int64_t *seq_offsets_host, int n_seqs,
                                 uint32_t *digests_dev, void *stream) {
    BSW_REQUIRE(digests_dev, "bsw_block_digests: null pointer");
    std::vector<int64_t> tab;
    int64_t total = 0;
    if (int rc = bd_table(blocks_dev, channels, n_slots, block_host, seq_offsets_host, n_seqs, tab, total)) return rc;
    return bd_run(tab, blocks_dev, extents_dev, channels, n_slots, n_seqs, digests_dev, nullptr, nullptr,
                  (cudaStream_t)stream);
}

extern "C" int bsw_block_digests_check(const uint8_t *blocks_dev, const int16_t *extents_dev, int channels,
                                       int64_t n_slots, const int64_t *block_host, const int64_t *seq_offsets_host,
                                       int n_seqs, const uint32_t *expected_dev, int64_t *result_dev, void *stream) {
    BSW_REQUIRE(expected_dev && result_dev, "bsw_block_digests_check: null pointer");
    std::vector<int64_t> tab;
    int64_t total = 0;
    if (int rc = bd_table(blocks_dev, channels, n_slots, block_host, seq_offsets_host, n_seqs, tab, total)) return rc;
    return bd_run(tab, blocks_dev, extents_dev, channels, n_slots, n_seqs, nullptr, expected_dev, result_dev,
                  (cudaStream_t)stream);
}
