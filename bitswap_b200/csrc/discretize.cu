// Sampling epilogue and bin fit of the latent-space discretisation (sm_90a).
//
// Reference: discretize() / discretize_kbins(), discretization.py:30-118.  Per latent level it draws 30 * 2^q samples per
// dimension from the generative chain and as many from the inference chain,
//     z = mu + scale * eps,   eps = log(u) - log(1 - u),  u ~ U(0,1) clamped to [bound, 1 - bound]
// (utils/torch/rand.py:11-20,22-29), stores them as float16 (:59-61), and fits 2^q equal-width bins per dimension between
// the extrema of the float16 samples (KBinsDiscretizer 'uniform' == np.linspace(min, max, 2^q + 1), :105-118).
//
//   k_sample_logistic   one pass over a [rows, dim] batch of (mu, scale, u): writes the float16 samples the next net reads
//                       and folds them into per-dimension running extrema -- the reference's 2 * 30 * 2^q * zdim float16
//                       sample matrix per level never has to be re-read for the fit.
//   k_uniform_edges     extrema -> float64 endpoints / centres with np.linspace's arithmetic (start + k * step, last
//                       point forced to stop), written straight into the Bins table layout.
// The uniforms are an input (torch's generator on the device): the test feeds identical noise to a torch-CPU run of the same nets.
#include <cuda_fp16.h>
#include <string.h>
#include "bsw_common.cuh"

namespace {

// order-preserving float <-> uint32 map, so that extrema are integer atomics
__device__ __forceinline__ uint32_t f2ord(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

constexpr int SR = 64;       // rows per CTA strip

__global__ void k_minmax_reset(uint32_t *__restrict__ mm, int dim) {
    int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d < dim) { mm[d] = 0xffffffffu; mm[dim + d] = 0u; }          // min slot, max slot
}

__global__ void k_sample_logistic(const float *__restrict__ mu, const float *__restrict__ sc, int64_t sc_row_stride,
                                  const float *__restrict__ u, float bound, __half *__restrict__ out,
                                  uint32_t *__restrict__ mm, int64_t rows, int dim) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;             // consecutive threads -> consecutive dimensions
    if (d >= dim) return;
    const int64_t r0 = (int64_t)blockIdx.y * SR, r1 = min(rows, r0 + SR);
    float lo = __int_as_float(0x7f800000), hi = __int_as_float(0xff800000);
    for (int64_t r = r0; r < r1; ++r) {
        const int64_t i = r * dim + d;
        float uu = fminf(fmaxf(u[i], bound), 1.0f - bound);          // rand.py:15
        const float eps = logf(uu) - log1pf(-uu);                    // rand.py:16-17 (logistic_eps)
        // rand.py:6-8 mu + scale * eps: the compressing-mode nets hand out float64 (cifar_train.py:375-376 up-cast), so
        // the reference forms the sample in float64 and rounds ONCE, float64 -> float16 (discretization.py:59-61,68)
        const double z = __dadd_rn((double)mu[i], __dmul_rn((double)sc[r * sc_row_stride + d], (double)eps));
        const __half h = __double2half(z);
        out[i] = h;
        const float zf = __half2float(h);
        lo = fminf(lo, zf); hi = fmaxf(hi, zf);
    }
    if (r1 > r0) {
        atomicMin(mm + d, f2ord(lo));
        atomicMax(mm + dim + d, f2ord(hi));
    }
}

// float16 samples produced elsewhere (e.g. the top-level prior draw): fold into the extrema
__global__ void k_minmax_half(const __half *__restrict__ s, uint32_t *__restrict__ mm, int64_t rows, int dim) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= dim) return;
    const int64_t r0 = (int64_t)blockIdx.y * SR, r1 = min(rows, r0 + SR);
    float lo = __int_as_float(0x7f800000), hi = __int_as_float(0xff800000);
    for (int64_t r = r0; r < r1; ++r) {
        const float zf = __half2float(s[r * dim + d]);
        lo = fminf(lo, zf); hi = fmaxf(hi, zf);
    }
    if (r1 > r0) {
        atomicMin(mm + d, f2ord(lo));
        atomicMax(mm + dim + d, f2ord(hi));
    }
}

// np.linspace(lo, hi, n + 1): step = (hi - lo) / n, y_k = lo + k * step, y_n = hi; endpoints = y_1..y_{n-1},
// centres = (y_k + y_{k+1}) / 2 (discretization.py:112-117)
__global__ void k_uniform_edges(const uint32_t *__restrict__ mm, int dim, int n, double *__restrict__ endp, int64_t endp_row_stride,
                                double *__restrict__ cen, int64_t cen_row_stride) {
    const int d = blockIdx.y;
    const double lo = (double)ord2f(mm[d]), hi = (double)ord2f(mm[dim + d]);
    const double step = (hi - lo) / (double)n;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const double y0 = lo + (double)k * step;
        const double y1 = (k + 1 == n) ? hi : lo + (double)(k + 1) * step;
        if (k >= 1) endp[d * endp_row_stride + k - 1] = y0;
        cen[d * cen_row_stride + k] = (y0 + y1) / 2;
    }
}

}  // namespace

extern "C" int bsw_discretize_reset(uint32_t *minmax_dev, int dim, void *stream) {
    BSW_REQUIRE(minmax_dev && dim > 0, "bsw_discretize_reset: bad arguments");
    k_minmax_reset<<<(dim + 255) / 256, 256, 0, (cudaStream_t)stream>>>(minmax_dev, dim);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

extern "C" int bsw_discretize_sample(const float *mu_dev, const float *scale_dev, int64_t scale_row_stride, const float *u_dev,
                                     float bound, void *out_half_dev, uint32_t *minmax_dev, int64_t rows, int dim, void *stream) {
    BSW_REQUIRE(mu_dev && scale_dev && u_dev && out_half_dev && minmax_dev && rows > 0 && dim > 0, "bsw_discretize_sample: bad arguments");
    BSW_REQUIRE(scale_row_stride == 0 || scale_row_stride >= dim, "bsw_discretize_sample: scale row stride");
    BSW_REQUIRE(bound > 0.f && bound < 0.5f, "bsw_discretize_sample: bound must lie in (0, 0.5)");
    dim3 grid((dim + 127) / 128, (unsigned)((rows + SR - 1) / SR));
    k_sample_logistic<<<grid, 128, 0, (cudaStream_t)stream>>>(mu_dev, scale_dev, scale_row_stride, u_dev, bound, (__half *)out_half_dev,
                                                             minmax_dev, rows, dim);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

extern "C" int bsw_discretize_fold(const void *samples_half_dev, uint32_t *minmax_dev, int64_t rows, int dim, void *stream) {
    BSW_REQUIRE(samples_half_dev && minmax_dev && rows > 0 && dim > 0, "bsw_discretize_fold: bad arguments");
    dim3 grid((dim + 127) / 128, (unsigned)((rows + SR - 1) / SR));
    k_minmax_half<<<grid, 128, 0, (cudaStream_t)stream>>>((const __half *)samples_half_dev, minmax_dev, rows, dim);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

extern "C" int bsw_discretize_edges(const uint32_t *minmax_dev, int dim, int quantbits, double *endpoints_dev, int64_t endp_row_stride,
                                    double *centres_dev, int64_t cen_row_stride, void *stream) {
    BSW_REQUIRE(minmax_dev && endpoints_dev && centres_dev && dim > 0 && quantbits >= 1 && quantbits <= 12, "bsw_discretize_edges: bad arguments");
    const int n = 1 << quantbits;
    BSW_REQUIRE(endp_row_stride >= n - 1 && cen_row_stride >= n, "bsw_discretize_edges: row strides");
    dim3 grid((n + 255) / 256, dim);
    k_uniform_edges<<<grid, 256, 0, (cudaStream_t)stream>>>(minmax_dev, dim, n, endpoints_dev, endp_row_stride, centres_dev, cen_row_stride);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}
