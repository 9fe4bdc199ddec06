// Device digests of the buffers that decide a bitstream: the folded model and the bin tables (include/bitswap_b200.h,
// bsw_digest).  Bins at quantbits 12 take 1.07 GB, which is why the words are hashed where they live.  Integer operations
// only, in a fixed order per chunk and across chunks, so the result does not depend on the launch shape or the device.
// Meant to catch accidental mismatches, not tampering: nothing here is cryptographic.
#include <stdint.h>
#include <vector>
#include "nets.cuh"

namespace {
constexpr int64_t DG_CHUNK = 8192;              // words per chunk
constexpr int DG_WARPS = 8;                     // chunks (warps) per CTA
constexpr uint64_t DG_PA = 0x9E3779B97F4A7C15ull, DG_PB = 0xC2B2AE3D27D4EB4Full;
constexpr uint64_t DG_CA = 0x5354414D50484131ull, DG_CB = 0x5354414D50484232ull;
constexpr uint64_t DG_DA = 0x4449474553544131ull, DG_DB = 0x4449474553544232ull;

__host__ __device__ __forceinline__ uint64_t dg_mix(uint64_t z) {       // splitmix64 finaliser (a bijection)
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t dg_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

// One warp per chunk: lane l mixes words l, l + 32, ... of the chunk (coalesced), then lane states are folded in lane
// order.  out: [nchunks][2] (ha, hb).
__global__ void __launch_bounds__(32 * DG_WARPS) k_digest_chunks(const uint8_t *__restrict__ p, int64_t bytes,
                                                                  int64_t nchunks, uint64_t *__restrict__ out) {
    const int64_t c = (int64_t)blockIdx.x * DG_WARPS + threadIdx.x / 32;
    const int lane = threadIdx.x & 31;
    if (c >= nchunks) return;                                            // warp-uniform
    const int64_t nw = (bytes + 7) / 8, full = bytes / 8, w0 = c * DG_CHUNK;
    const int64_t len = nw - w0 < DG_CHUNK ? nw - w0 : DG_CHUNK;
    const uint64_t *q = reinterpret_cast<const uint64_t *>(p);
    uint64_t a = dg_mix(((uint64_t)c << 6) | (uint64_t)(2 * lane)), b = dg_mix(((uint64_t)c << 6) | (uint64_t)(2 * lane + 1));
    for (int64_t i = lane; i < len; i += 32) {
        const int64_t g = w0 + i;
        uint64_t w = 0;
        if (g < full) {
            w = __ldg(q + g);
        } else {                                                         // the last, partial word: zero-padded
            for (int k = 0; k < (int)(bytes - 8 * g); ++k) w |= (uint64_t)p[8 * g + k] << (8 * k);
        }
        a = dg_rotl(a ^ w, 29) * DG_PA;
        b = (dg_rotl(b, 23) + w) * DG_PB;
    }
    uint64_t ha = dg_mix((uint64_t)c ^ DG_CA), hb = dg_mix((uint64_t)c + DG_CB);
    for (int l = 0; l < 32; ++l) {
        ha = dg_mix(ha ^ __shfl_sync(0xffffffffu, a, l));
        hb = dg_mix(hb + __shfl_sync(0xffffffffu, b, l));
    }
    if (lane == 0) { out[2 * c] = ha; out[2 * c + 1] = hb; }
}

int digest_dev(const void *dev, int64_t bytes, uint32_t out4[4], cudaStream_t st) {
    const int64_t nchunks = ((bytes + 7) / 8 + DG_CHUNK - 1) / DG_CHUNK;
    std::vector<uint64_t> h(2 * nchunks);
    if (nchunks) {
        uint64_t *d = nullptr;
        BSW_CUDA(cudaMalloc(&d, sizeof(uint64_t) * 2 * nchunks));
        k_digest_chunks<<<(unsigned)((nchunks + DG_WARPS - 1) / DG_WARPS), 32 * DG_WARPS, 0, st>>>(
            (const uint8_t *)dev, bytes, nchunks, d);
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(h.data(), d, sizeof(uint64_t) * 2 * nchunks, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cudaFree(d);
        BSW_CUDA(e);
    }
    uint64_t da = dg_mix((uint64_t)bytes ^ DG_DA), db = dg_mix((uint64_t)bytes + DG_DB);
    for (int64_t c = 0; c < nchunks; ++c) {
        da = dg_mix(da ^ h[2 * c]);
        db = dg_mix(db + h[2 * c + 1]);
    }
    out4[0] = (uint32_t)da; out4[1] = (uint32_t)(da >> 32); out4[2] = (uint32_t)db; out4[3] = (uint32_t)(db >> 32);
    return BSW_OK;
}

// A record of host words (sizes, shapes and the digests of device buffers), digested as one buffer.
struct Record {
    std::vector<uint32_t> w;
    void add(int64_t v) { w.push_back((uint32_t)v); }
    int add_digest(const void *dev, int64_t bytes, cudaStream_t st) {
        uint32_t d[4];
        if (int rc = digest_dev(dev, bytes, d, st)) return rc;
        w.insert(w.end(), d, d + 4);
        return BSW_OK;
    }
    int finish(uint32_t out4[4], cudaStream_t st) {
        void *d = nullptr;
        BSW_CUDA(cudaMalloc(&d, sizeof(uint32_t) * w.size()));
        cudaError_t e = cudaMemcpyAsync(d, w.data(), sizeof(uint32_t) * w.size(), cudaMemcpyHostToDevice, st);
        int rc = e == cudaSuccess ? digest_dev(d, (int64_t)(sizeof(uint32_t) * w.size()), out4, st) : BSW_OK;
        cudaFree(d);
        BSW_CUDA(e);
        return rc;
    }
};
}  // namespace

extern "C" int bsw_bitstream_revision(void) { return BSW_BITSTREAM_REVISION; }

extern "C" int bsw_digest(const void *dev, int64_t bytes, uint32_t out4[4], void *stream) {
    BSW_REQUIRE(out4 && bytes >= 0 && (dev || bytes == 0), "bsw_digest: bad arguments");
    BSW_REQUIRE(((uintptr_t)dev & 7) == 0, "bsw_digest: the buffer must be 8-byte aligned");
    return digest_dev(dev, bytes, out4, (cudaStream_t)stream);
}

extern "C" int bsw_model_digest(bsw_model *m, uint32_t out4[4], void *stream) {
    BSW_REQUIRE(m && out4, "bsw_model_digest: null argument");
    BSW_REQUIRE(m->finalized, "bsw_model_digest: model not finalized");
    if (!m->digest_ok) {
        cudaStream_t st = (cudaStream_t)stream;
        const bsw_model_desc &d = m->d;
        Record r;
        for (int32_t v : {d.xc, d.nz, d.zchannels, d.nprocessing, d.kernel_size, d.resdepth, d.reswidth, d.cond_xscale}) r.add(v);
        r.add((int64_t)m->convs.size());
        for (const ConvSlot &c : m->convs) {
            for (int v : {c.Cin, c.Cout, c.ks, c.CinP, c.CoutP, c.parts}) r.add(v);
            if (int rc = r.add_digest(c.w, (int64_t)sizeof(float) * c.ks * c.ks * c.CinP * c.CoutP, st)) return rc;
            if (int rc = r.add_digest(c.bias, (int64_t)sizeof(float) * c.CoutP, st)) return rc;
        }
        if (!d.cond_xscale) {
            r.add(m->xdim);
            if (int rc = r.add_digest(m->xscale, (int64_t)sizeof(float) * m->xdim, st)) return rc;
        }
        if (int rc = r.finish(m->digest, st)) return rc;
        m->digest_ok = true;
    }
    for (int i = 0; i < 4; ++i) out4[i] = m->digest[i];
    return BSW_OK;
}

extern "C" int bsw_bins_digest(bsw_bins *b, uint32_t out4[4], void *stream) {
    BSW_REQUIRE(b && out4, "bsw_bins_digest: null argument");
    if (!b->digest_ok) {
        cudaStream_t st = (cudaStream_t)stream;
        const int64_t zbytes = (int64_t)sizeof(double) * b->nz * b->zdim * b->S;
        Record r;
        r.add(b->q); r.add(b->nz); r.add(b->zdim);
        if (int rc = r.add_digest(b->zend, zbytes, st)) return rc;
        if (int rc = r.add_digest(b->zcen, zbytes, st)) return rc;
        if (int rc = r.add_digest(b->xend, (int64_t)sizeof(double) * 256, st)) return rc;
        if (int rc = r.finish(b->digest, st)) return rc;
        b->digest_ok = true;
    }
    for (int i = 0; i < 4; ++i) out4[i] = b->digest[i];
    return BSW_OK;
}
