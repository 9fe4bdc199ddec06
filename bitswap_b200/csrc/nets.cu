// The inference-time hierarchical VAE (sm_90a): weight-norm folding, conv stacks, mu/sigma heads.
//
// Reference being replaced (fhkingma/bitswap @ dfe0bf7d):
//   Model.infer(i)(given) / Model.generate(i)(given), compressing mode   model/cifar_train.py:315-438
//   conditional x-scale head                                            model/imagenetcrop_train.py:306-315,417
//   WnConv2d._forward (weight norm)                                      utils/torch/modules.py:98-106
//   ResNetLayer.forward  x + conv2(ELU(conv1(ELU(x))))                   utils/torch/modules.py:229-241
//   Squeeze2d / UnSqueeze2d                                              utils/torch/modules.py:175-208
//
// Layout: hidden activations are NHWC float32 [n, 16*16, Wp] with the width padded to a multiple of
// 64 (252 -> 256); padded channels carry exact zeros (zero weights, zero bias, ELU(0) = 0).  Weight
// normalisation is folded once at load.  Every conv is one kernel with a fused epilogue: bias,
// residual add, ELU (once or twice, see RunPlan), and for the heads the sigmoid/softplus scale
// transforms and the (Un)Squeeze2d index maps, so mu/sigma leave the net already in the flat CHW
// order the coder consumes.
//
// This file holds the float32 SIMT implicit-GEMM conv (k_conv_simt): the permanent path for the
// small-contraction convs (in-convs with 1..12 input channels, mu/sigma heads with <= 32 outputs) and
// the fallback-free baseline for the dense W->W convs; conv_tc.cu adds the wgmma tensor-core path for those.
#include <math.h>
#include <map>
#include <string>
#include <vector>
#include "bsw_common.cuh"
#include "nets.cuh"

// ------------------------------------------------------------------------------------------------
// device math
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }                 // nn.ELU(alpha=1)
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float softplusf_(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }   // -logsigmoid(-x), modules.py:112-114

__device__ __forceinline__ float scale_transform(float r, int kind) {
    switch (kind) {
        case SCALE_INFER:   return 0.1f + 0.9f * sigmoidf_(r + 2.f);                               // cifar_train.py:349,368
        case SCALE_DEEPGEN: return 0.1f + 0.9f * softplusf_(r + 0.54132485461291810f);             // :426  log(e-1)
        case SCALE_X:       return ((2.f / 255.f) / 8.f) + softplusf_(r);                          // :411 / imagenetcrop :417
    }
    return r;
}

// ------------------------------------------------------------------------------------------------
// float32 SIMT conv: implicit GEMM, M = 256 pixels of one image, N = COT output channels per CTA,
// K = taps x input channels in chunks of 8.  256 threads; thread (cog = t%8, pg = t/8) owns an
// 8-pixel row segment x TCO output channels.
// ------------------------------------------------------------------------------------------------
constexpr int CC = 8;          // input channels per shared-memory chunk
// padded row stride of the input patch (floats): at least its 16 + KS - 1 columns, a multiple of 4 for the float4 row loads
template <int KS> constexpr int IWS_OF = KS <= 5 ? 20 : 24;

// Shared memory: [CC][IH][IWS] input patch + [KS^2][CC][COT] weights.  KS = 7, TCO = 8: 16.5 KB + 98 KB = 114.5 KB, so
// one CTA per SM (the KS <= 5 instantiations keep two); KS = 7, TCO = 2: 41 KB.
template <int KS, int TCO>
__global__ void __launch_bounds__(256, 2) k_conv_simt(ConvArgs a) {
    constexpr int R = KS / 2, IH = 16 + KS - 1, COT = 8 * TCO, TAPS = KS * KS, IWS = IWS_OF<KS>;
    extern __shared__ float sm[];
    float *in_s = sm;                               // [CC][IH][IWS]
    float *w_s = sm + CC * IH * IWS;                // [TAPS][CC][COT]
    const int n = blockIdx.x, co0 = blockIdx.y * COT;
    const int t = threadIdx.x, cog = t & 7, pg = t >> 3, prow = pg >> 1, pcol0 = (pg & 1) * 8;

    float acc[8][TCO];
#pragma unroll
    for (int p = 0; p < 8; ++p)
#pragma unroll
        for (int c = 0; c < TCO; ++c) acc[p][c] = 0.f;

    for (int c0 = 0; c0 < a.CinP; c0 += CC) {
        __syncthreads();
        // ---- stage the input patch (zero padded halo) -------------------------------------------
        if (a.in_mode == IN_NHWC) {
            const float *src = a.in + (int64_t)n * 256 * a.ld_in + c0;
            for (int pos = t; pos < IH * IH; pos += 256) {
                int y = pos / IH, x = pos - y * IH;
                int iy = y - R, ix = x - R;
                float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
                if (iy >= 0 && iy < 16 && ix >= 0 && ix < 16) {
                    const float4 *p = reinterpret_cast<const float4 *>(src + (int64_t)(iy * 16 + ix) * a.ld_in);
                    v0 = __ldg(p);
                    v1 = __ldg(p + 1);
                }
                float *d = in_s + y * IWS + x;
                d[0 * IH * IWS] = v0.x; d[1 * IH * IWS] = v0.y; d[2 * IH * IWS] = v0.z; d[3 * IH * IWS] = v0.w;
                d[4 * IH * IWS] = v1.x; d[5 * IH * IWS] = v1.y; d[6 * IH * IWS] = v1.z; d[7 * IH * IWS] = v1.w;
            }
        } else {
            // flat CHW `given` (cifar_train.py:330,355,393); IN_CHW_X applies Squeeze2d(2) on the fly:
            // channel c*4 + fh*2 + fw  <-  pixel (2h+fh, 2w+fw) of image channel c  (modules.py:183-185)
            const float *src = a.in + (int64_t)n * a.in_dim;
            for (int idx = t; idx < CC * IH * IH; idx += 256) {
                int ci = idx / (IH * IH), pos = idx - ci * (IH * IH);
                int y = pos / IH, x = pos - y * IH;
                int iy = y - R, ix = x - R, ch = c0 + ci;
                float v = 0.f;
                if (ch < a.Cin && iy >= 0 && iy < 16 && ix >= 0 && ix < 16) {
                    if (a.in_mode == IN_CHW_Z) v = __ldg(src + ch * 256 + iy * 16 + ix);
                    else v = __ldg(src + (ch >> 2) * 1024 + (2 * iy + ((ch >> 1) & 1)) * 32 + 2 * ix + (ch & 1));
                }
                in_s[(ci * IH + y) * IWS + x] = v;
            }
        }
        // ---- stage the weight chunk [TAPS][CC][COT] from [TAPS][CinP][CoutP] -------------------------
        for (int idx = t; idx < TAPS * CC * COT / 4; idx += 256) {
            int co4 = idx % (COT / 4), rest = idx / (COT / 4);
            int ci = rest % CC, tap = rest / CC;
            const float4 *p = reinterpret_cast<const float4 *>(a.w + ((int64_t)tap * a.CinP + c0 + ci) * a.CoutP + co0) + co4;
            reinterpret_cast<float4 *>(w_s)[idx] = __ldg(p);
        }
        __syncthreads();
        // ---- multiply-accumulate ----------------------------------------------------------------------
#pragma unroll 1
        for (int ci = 0; ci < CC; ++ci) {
#pragma unroll
            for (int dy = 0; dy < KS; ++dy) {
                const float *rp = in_s + (ci * IH + prow + dy) * IWS + pcol0;
                // the 8 + KS - 1 patch values this row of taps reads: float4 loads, then a float2 tail (KS = 3, 7)
                constexpr int NV = 8 + KS - 1, NV4 = NV / 4 * 4;
                float iv[NV];
#pragma unroll
                for (int v4 = 0; v4 < NV / 4; ++v4) {
                    float4 q4 = *reinterpret_cast<const float4 *>(rp + 4 * v4);
                    iv[4 * v4] = q4.x; iv[4 * v4 + 1] = q4.y; iv[4 * v4 + 2] = q4.z; iv[4 * v4 + 3] = q4.w;
                }
                if constexpr (NV % 4 == 2) {
                    float2 q2 = *reinterpret_cast<const float2 *>(rp + NV4);
                    iv[NV4] = q2.x; iv[NV4 + 1] = q2.y;
                }
#pragma unroll
                for (int dx = 0; dx < KS; ++dx) {
                    const float *wp = w_s + ((dy * KS + dx) * CC + ci) * COT + cog * TCO;
                    float wv[TCO];
                    if constexpr (TCO == 8) {
                        float4 w0 = *reinterpret_cast<const float4 *>(wp), w1 = *reinterpret_cast<const float4 *>(wp + 4);
                        wv[0] = w0.x; wv[1] = w0.y; wv[2] = w0.z; wv[3] = w0.w;
                        wv[4] = w1.x; wv[5] = w1.y; wv[6] = w1.z; wv[7] = w1.w;
                    } else {
                        float2 w0 = *reinterpret_cast<const float2 *>(wp);
                        wv[0] = w0.x; wv[1] = w0.y;
                    }
#pragma unroll
                    for (int p = 0; p < 8; ++p)
#pragma unroll
                        for (int c = 0; c < TCO; ++c) acc[p][c] = fmaf(iv[p + dx], wv[c], acc[p][c]);
                }
            }
        }
    }

    // ---- epilogue ----------------------------------------------------------------------------------------
    float bias[TCO];
#pragma unroll
    for (int c = 0; c < TCO; ++c) bias[c] = a.bias[co0 + cog * TCO + c];

    if (a.out_mode == OUT_NHWC) {
#pragma unroll
        for (int p = 0; p < 8; ++p) {
            int px = prow * 16 + pcol0 + p;
            int64_t off = ((int64_t)n * 256 + px) * a.CoutP + co0 + cog * TCO;
            float r[TCO];
#pragma unroll
            for (int c = 0; c < TCO; ++c) r[c] = acc[p][c] + bias[c];
            if (a.resid) {
#pragma unroll
                for (int c = 0; c < TCO; ++c) r[c] += a.resid[off + c];          // x + conv2(...)  modules.py:241
            }
            if (a.T_elu) {
#pragma unroll
                for (int c = 0; c < TCO; ++c) r[c] = elu1(r[c]);
            }
            if (a.T) {
#pragma unroll
                for (int c = 0; c < TCO; ++c) a.T[off + c] = r[c];
            }
            if (a.A) {
#pragma unroll
                for (int c = 0; c < TCO; ++c) a.A[off + c] = a.A_elu ? elu1(r[c]) : r[c];
            }
        }
    } else {
        // heads: channels [0, n_mu) are mu, [n_mu, n_mu+n_sc) the pre-activation of the scale
#pragma unroll
        for (int c = 0; c < TCO; ++c) {
            int co = co0 + cog * TCO + c;
            bool is_mu = co < a.n_mu;
            int o = is_mu ? co : co - a.n_mu;
            if (!is_mu && o >= a.n_sc) continue;
            float *dst = (is_mu ? a.mu : a.scale) + (int64_t)n * a.out_dim;
#pragma unroll
            for (int p = 0; p < 8; ++p) {
                float r = acc[p][c] + bias[c];
                if (!is_mu) r = scale_transform(r, a.scale_kind);
                int y = prow, x = pcol0 + p;
                if (a.out_mode == OUT_HEAD_Z) dst[o * 256 + y * 16 + x] = r;
                else                                                                      // UnSqueeze2d, modules.py:205-207
                    dst[(o >> 2) * 1024 + (2 * y + ((o >> 1) & 1)) * 32 + 2 * x + (o & 1)] = r;
            }
        }
    }
}

template <int KS, int TCO>
static int launch_conv_simt(const ConvArgs &a, int64_t n, cudaStream_t st) {
    constexpr int IH = 16 + KS - 1, COT = 8 * TCO;
    size_t smem = sizeof(float) * (CC * IH * IWS_OF<KS> + KS * KS * CC * COT);
    static bool attr_done = false;
    if (!attr_done) {
        BSW_CUDA(cudaFuncSetAttribute(k_conv_simt<KS, TCO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        bsw_prefer_max_shared(k_conv_simt<KS, TCO>);       // same L1/shared split as every other kernel of the path
        attr_done = true;
    }
    dim3 grid((unsigned)n, a.CoutP / COT);
    k_conv_simt<KS, TCO><<<grid, 256, smem, st>>>(a);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

int bsw_conv_simt(const ConvArgs &a, int ks, int64_t n, cudaStream_t st) {
    bool wide = (a.CoutP % 64) == 0;
    if (ks == 5) return wide ? launch_conv_simt<5, 8>(a, n, st) : launch_conv_simt<5, 2>(a, n, st);
    if (ks == 3) return wide ? launch_conv_simt<3, 8>(a, n, st) : launch_conv_simt<3, 2>(a, n, st);
    if (ks == 1) return wide ? launch_conv_simt<1, 8>(a, n, st) : launch_conv_simt<1, 2>(a, n, st);
    if (ks == 7) return wide ? launch_conv_simt<7, 8>(a, n, st) : launch_conv_simt<7, 2>(a, n, st);
    bsw_set_error("conv kernel size %d not supported (1, 3, 5 or 7)", ks);
    return BSW_E_INVALID;
}

// ------------------------------------------------------------------------------------------------
// Model: conv slots, name map, run plans
// ------------------------------------------------------------------------------------------------
static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

static int add_conv(bsw_model *m, const std::string &name, int Cin, int Cout, int ks, int cout_tile) {
    ConvSlot s;
    s.name = name;
    s.Cin = Cin; s.Cout = Cout; s.ks = ks;
    s.CinP = round_up(Cin, CC);
    s.CoutP = round_up(Cout, cout_tile);
    s.w = nullptr; s.bias = nullptr;
    s.loaded_mask = 0; s.parts = 1;
    m->convs.push_back(s);
    return (int)m->convs.size() - 1;
}

static void add_block(bsw_model *m, NetPlan &np, const std::string &prefix, int ks, int nlayers) {
    if (nlayers <= 0) return;
    const int W = m->d.reswidth, Wp = m->Wp;
    BlockPlan bp;
    for (int l = 1; l <= nlayers; ++l) {
        std::string p = prefix + ".res" + std::to_string(W) + "layer" + std::to_string(l);
        int c1 = add_conv(m, p + ".conv1", W, W, ks, 64), c2 = add_conv(m, p + ".conv2", W, W, ks, 64);
        m->convs[c1].CinP = m->convs[c2].CinP = Wp;      // hidden tensors are Wp wide
        m->names[p + ".conv1"] = {c1, 0};
        m->names[p + ".conv2"] = {c2, 0};
        bp.layers.push_back({c1, c2});
    }
    np.blocks.push_back(bp);
}

extern "C" int bsw_model_create(bsw_model **out, const bsw_model_desc *d) {
    BSW_REQUIRE(out && d, "bsw_model_create: null argument");
    BSW_REQUIRE(d->nz >= 1 && d->xc >= 1 && d->zchannels >= 1 && d->reswidth >= 1 && d->nprocessing >= 0 &&
                d->resdepth >= 0 && d->max_batch >= 1, "bsw_model_create: bad descriptor");
    BSW_REQUIRE(d->kernel_size == 1 || d->kernel_size == 3 || d->kernel_size == 5 || d->kernel_size == 7,
                "bsw_model_create: kernel_size must be 1, 3, 5 or 7");
    bsw_model *m = new bsw_model();
    m->d = *d;
    m->Wp = round_up(d->reswidth, 64);
    m->zdim = d->zchannels * 256;
    m->xdim = d->xc * 1024;
    // ks: the reference's self.kernel_size (ResNet blocks res1 / deep*_res, z in-convs, heads); infer_in and the
    // nprocessing blocks are 5x5 whatever it is (padding_proc, cifar_train.py:45-47)
    const int W = d->reswidth, zc = d->zchannels, C = d->xc, nz = d->nz, ks = d->kernel_size;
    std::vector<int> rd(nz, 0);                        // model/cifar_train.py:66-72
    for (int r = 0, i = 0; r < d->resdepth; ++r) { if (i == nz) i = 0; rd[i++]++; }

    m->infer.resize(nz);
    m->gen.resize(nz);
    // ---- infer(0): cifar_train.py:89-141, 336-349
    {
        NetPlan &np = m->infer[0];
        np.in_conv = add_conv(m, "infer_in.1", 4 * C, W, 5, 64);
        m->names["infer_in.1"] = {np.in_conv, 0};
        np.in_mode = IN_CHW_X; np.in_dim = m->xdim;
        add_block(m, np, "infer_res0.0", 5, d->nprocessing);
        add_block(m, np, "infer_res1.0", ks, rd[0]);
        np.head = add_conv(m, "infer_mu|infer_std", W, 2 * zc, ks, 16);
        m->convs[np.head].CinP = m->Wp; m->convs[np.head].parts = 2;
        m->names["infer_mu"] = {np.head, 0};
        m->names["infer_std"] = {np.head, zc};
        np.out_mode = OUT_HEAD_Z; np.n_mu = zc; np.n_sc = zc; np.scale_kind = SCALE_INFER; np.out_dim = m->zdim;
    }
    // ---- infer(i>0) / generate(i>0): cifar_train.py:143-245, 352-368, 414-426
    for (int kind = 0; kind < 2; ++kind) {
        const std::string nm = kind == 0 ? "deepinfer" : "deepgen";
        for (int j = 0; j + 1 < nz; ++j) {
            NetPlan &np = kind == 0 ? m->infer[j + 1] : m->gen[j + 1];
            std::string js = std::to_string(j);
            np.in_conv = add_conv(m, nm + "_in." + js + ".0", zc, W, ks, 64);
            m->names[nm + "_in." + js + ".0"] = {np.in_conv, 0};
            np.in_mode = IN_CHW_Z; np.in_dim = m->zdim;
            add_block(m, np, nm + "_res." + js + ".0", ks, rd[j + 1]);
            np.head = add_conv(m, nm + "_mu|std." + js, W, 2 * zc, ks, 16);
            m->convs[np.head].CinP = m->Wp; m->convs[np.head].parts = 2;
            m->names[nm + "_mu." + js + ".0"] = {np.head, 0};
            m->names[nm + "_std." + js + ".0"] = {np.head, zc};
            np.out_mode = OUT_HEAD_Z; np.n_mu = zc; np.n_sc = zc; np.out_dim = m->zdim;
            np.scale_kind = kind == 0 ? SCALE_INFER : SCALE_DEEPGEN;
        }
    }
    // ---- generate(0): cifar_train.py:247-308, 396-411
    {
        NetPlan &np = m->gen[0];
        np.in_conv = add_conv(m, "gen_in.0", zc, W, ks, 64);
        m->names["gen_in.0"] = {np.in_conv, 0};
        np.in_mode = IN_CHW_Z; np.in_dim = m->zdim;
        add_block(m, np, "gen_res1.0", ks, rd[0]);
        add_block(m, np, "gen_res0.0", 5, d->nprocessing);
        int nh = d->cond_xscale ? 8 * C : 4 * C;
        np.head = add_conv(m, "gen_mu.0|gen_std.0", W, nh, ks, 16);
        m->convs[np.head].CinP = m->Wp; m->convs[np.head].parts = d->cond_xscale ? 2 : 1;
        m->names["gen_mu.0"] = {np.head, 0};
        if (d->cond_xscale) m->names["gen_std.0"] = {np.head, 4 * C};
        np.out_mode = OUT_HEAD_X; np.n_mu = 4 * C; np.n_sc = d->cond_xscale ? 4 * C : 0; np.scale_kind = SCALE_X;
        np.out_dim = m->xdim;
    }
    // ---- activations: one trunk + two ping-pong conv-input buffers, [max_batch, 256, Wp] float32
    size_t act = (size_t)d->max_batch * 256 * m->Wp * sizeof(float);
    BSW_CUDA(cudaMalloc(&m->bufT, act));
    BSW_CUDA(cudaMalloc(&m->bufA, act));
    BSW_CUDA(cudaMalloc(&m->bufB, act));
    BSW_CUDA(cudaMalloc(&m->xscale, sizeof(float) * m->xdim));
    m->have_gen_std = false;
    m->finalized = false;
    *out = m;
    return BSW_OK;
}

extern "C" int bsw_model_destroy(bsw_model *m) {
    if (!m) return BSW_OK;
    for (auto &c : m->convs) { cudaFree(c.w); cudaFree(c.bias); }
    cudaFree(m->bufT); cudaFree(m->bufA); cudaFree(m->bufB); cudaFree(m->xscale);
    bsw_model_tc_release(m);
    delete m;
    return BSW_OK;
}

extern "C" int bsw_model_load_conv(bsw_model *m, const char *prefix, const float *v, const float *gain, const float *b,
                                   int O, int I, int k, int loggain) {
    BSW_REQUIRE(m && prefix && v && gain && b, "bsw_model_load_conv: null argument");
    auto it = m->names.find(prefix);
    if (it == m->names.end()) {
        bsw_set_error("bsw_model_load_conv: unknown conv '%s' for this model", prefix);
        return BSW_E_INVALID;
    }
    ConvSlot &s = m->convs[it->second.slot];
    int co_off = it->second.co_off;
    int expectO = s.parts == 2 ? s.Cout / 2 : s.Cout;
    if (O != expectO || I != s.Cin || k != s.ks) {
        bsw_set_error("bsw_model_load_conv: '%s' has shape [%d,%d,%d,%d], expected [%d,%d,%d,%d]", prefix, O, I, k, k,
                      expectO, s.Cin, s.ks, s.ks);
        return BSW_E_INVALID;
    }
    const int taps = k * k;
    if (!s.w) {
        BSW_CUDA(cudaMalloc(&s.w, sizeof(float) * taps * s.CinP * s.CoutP));
        BSW_CUDA(cudaMalloc(&s.bias, sizeof(float) * s.CoutP));
        BSW_CUDA(cudaMemset(s.w, 0, sizeof(float) * taps * s.CinP * s.CoutP));
        BSW_CUDA(cudaMemset(s.bias, 0, sizeof(float) * s.CoutP));
        s.host_w.assign((size_t)taps * s.CinP * s.CoutP, 0.f);
        s.host_b.assign(s.CoutP, 0.f);
    }
    // weight norm, folded once: w = v * (g / (||v|| + 1e-10)), g = softplus(gain) | gain   (modules.py:98-105)
    for (int o = 0; o < O; ++o) {
        double ss = 0.0;
        const float *vo = v + (size_t)o * I * taps;
        for (int e = 0; e < I * taps; ++e) ss += (double)vo[e] * (double)vo[e];
        float vnorm = (float)sqrt(ss);
        float g = gain[o];
        if (loggain) g = (float)(fmax((double)g, 0.0) + log1p(exp(-fabs((double)g))));
        float scale = g / (vnorm + 1e-10f);
        for (int i = 0; i < I; ++i)
            for (int tp = 0; tp < taps; ++tp)
                s.host_w[((size_t)tp * s.CinP + i) * s.CoutP + co_off + o] = vo[(size_t)i * taps + tp] * scale;
        s.host_b[co_off + o] = b[o];
    }
    BSW_CUDA(cudaMemcpy(s.w, s.host_w.data(), sizeof(float) * s.host_w.size(), cudaMemcpyHostToDevice));
    BSW_CUDA(cudaMemcpy(s.bias, s.host_b.data(), sizeof(float) * s.host_b.size(), cudaMemcpyHostToDevice));
    s.loaded_mask |= (co_off == 0) ? 1 : 2;
    m->digest_ok = false;
    return BSW_OK;
}

extern "C" int bsw_model_load_gen_std(bsw_model *m, const float *gen_std) {
    BSW_REQUIRE(m && gen_std, "bsw_model_load_gen_std: null argument");
    BSW_REQUIRE(!m->d.cond_xscale, "bsw_model_load_gen_std: this model has a conditional x-scale head");
    std::vector<float> sc(m->xdim);
    for (int i = 0; i < m->xdim; ++i) {       // (2/255)/8 + softplus(gen_std), cifar_train.py:411, in float32 like torch
        float g = gen_std[i];
        float sp = fmaxf(g, 0.f) + log1pf(expf(-fabsf(g)));
        sc[i] = ((2.f / 255.f) / 8.f) + sp;
    }
    BSW_CUDA(cudaMemcpy(m->xscale, sc.data(), sizeof(float) * m->xdim, cudaMemcpyHostToDevice));
    m->have_gen_std = true;
    m->digest_ok = false;
    return BSW_OK;
}

extern "C" int bsw_model_finalize(bsw_model *m) {
    BSW_REQUIRE(m, "null model");
    for (auto &c : m->convs) {
        int want = c.parts == 2 ? 3 : 1;
        if (c.loaded_mask != want) {
            bsw_set_error("bsw_model_finalize: conv '%s' not (fully) loaded", c.name.c_str());
            return BSW_E_INVALID;
        }
    }
    if (!m->d.cond_xscale && !m->have_gen_std) {
        bsw_set_error("bsw_model_finalize: gen_std not loaded");
        return BSW_E_INVALID;
    }
    if (m->d.use_tensor_cores) {
        if (int rc = bsw_model_tc_prepare(m)) return rc;
    }
    for (auto &c : m->convs) { c.host_w.clear(); c.host_w.shrink_to_fit(); }
    m->finalized = true;
    return BSW_OK;
}

extern "C" int bsw_model_set_tc_precision(bsw_model *m, int precision) {
    BSW_REQUIRE(m, "null model");
    BSW_REQUIRE(precision == BSW_TC_SPLIT || precision == BSW_TC_BF16,
                "bsw_model_set_tc_precision: BSW_TC_SPLIT (0) or BSW_TC_BF16 (1)");
    BSW_REQUIRE(m->d.use_tensor_cores, "bsw_model_set_tc_precision: a model without tensor cores has no tensor-core arithmetic");
    m->tc_precision = precision;        // read by every tensor-core launch; every net call writes the planes it reads
    return BSW_OK;
}

// ------------------------------------------------------------------------------------------------
// Running a net.  Value flow (h = trunk, all float32):
//   in-conv:            h = ELU(conv(given))                                   cifar_train.py:89-102 (Sequential(..., act))
//   per ResNet layer:   c1 = ELU(conv1(ELU(h))) ; h = h + conv2(c1)            modules.py:229-241
//   after each block:   h = ELU(h)                                             Sequential(ResNetBlock, act)
//   heads read h.
// Each conv kernel writes T (the new trunk, optionally ELU'd) and/or A (= T or ELU(T), the next conv's
// input), so every elementwise op lives in an epilogue.
// ------------------------------------------------------------------------------------------------
__global__ void k_broadcast_rows(const float *__restrict__ src, float *__restrict__ dst, int dim, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * dim) dst[i] = src[i % dim];
}

enum { ROLE_IN = 0, ROLE_DENSE = 1, ROLE_HEAD = 2 };

// Which path a net's convs take.  On the tensor-core path the dense convs read and write bf16 hi/lo planes, so the
// in-conv of a net with ResNet layers writes the first layer's planes (on the tensor cores, or SIMT + split when it has
// more than 32 input channels).  The head reads the planes the last ResNet conv wrote when it fits the tensor-core head
// (<= 32 outputs); otherwise it runs SIMT on the float32 trunk.
static bool net_on_tc(const bsw_model *m) { return m->d.use_tensor_cores && m->tc_ready; }
static bool in_writes_planes(const bsw_model *m, const NetPlan &np) { return net_on_tc(m) && !np.blocks.empty(); }
static bool head_on_tc(bsw_model *m, const NetPlan &np) {
    return in_writes_planes(m, np) && bsw_conv_tc_head_available(m, m->convs[np.head]);
}
// 1 if any net's head runs on the tensor cores (part of the codec fingerprint: BSW_TC_HEADS=0 changes mu/sigma)
int bsw_model_tc_heads(bsw_model *m) {
    for (const auto *nets : {&m->infer, &m->gen})
        for (const NetPlan &np : *nets)
            if (head_on_tc(m, np)) return 1;
    return 0;
}

// Runs one conv of net `np` in its role: the one place that picks its kernel(s).  `a` holds the input, the epilogue and,
// for the tensor-core kernels, the plane buffers read (in_planes) and written (A_planes).
static int dispatch_conv(bsw_model *m, const NetPlan &np, int role, const ConvSlot &c, ConvArgs a, int64_t n,
                         cudaStream_t st, int *launches) {
    if (role == ROLE_IN) {
        if (in_writes_planes(m, np) && c.tc_index >= 0) {
            // tensor-core in-conv: the trunk in float32, the first layer's input straight into the bf16 planes
            a.A = nullptr; a.A_planes = 0;
            return bsw_conv_tc_in(m, c, a, n, st, launches);
        }
        if (int rc = bsw_conv_simt(a, c.ks, n, st)) return rc;
        ++*launches;
        if (in_writes_planes(m, np)) {           // conv-input planes for the tensor-core layers: A -> bf16 hi/lo
            if (int rc = bsw_tc_split(m, a.A, 0, n, st)) return rc;
            ++*launches;
        }
        return BSW_OK;
    }
    const bool tc = role == ROLE_DENSE ? net_on_tc(m) : head_on_tc(m, np);
    int rc;
    if (!tc) rc = bsw_conv_simt(a, c.ks, n, st);
    else if (role == ROLE_DENSE) rc = bsw_conv_tc(m, c, a, n, st);
    else rc = bsw_conv_tc_head(m, c, a, n, st);
    if (rc) return rc;
    ++*launches;
    return BSW_OK;
}

static int run_net(bsw_model *m, const NetPlan &np, const float *given, int64_t n, float *mu, float *scale,
                   cudaStream_t st, int *launches, BswProf *prof) {
    BswProf noprof;
    if (!prof) prof = &noprof;
    BSW_REQUIRE(m->finalized, "model not finalized");
    BSW_REQUIRE(n >= 1 && n <= m->d.max_batch, "batch exceeds the model's max_batch");
    const int Wp = m->Wp;
    const bool has_blocks = !np.blocks.empty();
    // heads on the tensor cores: they read the trunk as bf16 planes, which the last ResNet conv then has to write
    const bool tc_head = head_on_tc(m, np);
    float *T = m->bufT, *A = m->bufA, *B = m->bufB;
    {   // in-conv
        const ConvSlot &c = m->convs[np.in_conv];
        ConvArgs a = {};
        a.in = given; a.in_mode = np.in_mode; a.in_dim = np.in_dim; a.Cin = c.Cin; a.CinP = c.CinP; a.ld_in = 0;
        a.w = c.w; a.bias = c.bias; a.CoutP = c.CoutP;
        a.out_mode = OUT_NHWC; a.T = T; a.T_elu = 1; a.A = has_blocks ? A : nullptr; a.A_elu = 1;
        prof->begin(CAT_CONV_IN, st);
        if (int rc = dispatch_conv(m, np, ROLE_IN, c, a, n, st, launches)) return rc;
        prof->end(st);
    }
    for (size_t bi = 0; bi < np.blocks.size(); ++bi) {
        const BlockPlan &bp = np.blocks[bi];
        for (size_t li = 0; li < bp.layers.size(); ++li) {
            const bool last_layer = li + 1 == bp.layers.size();
            const bool last_block = bi + 1 == np.blocks.size();
            for (int half = 0; half < 2; ++half) {
                const ConvSlot &c = m->convs[half == 0 ? bp.layers[li].first : bp.layers[li].second];
                ConvArgs a = {};
                a.in_mode = IN_NHWC; a.Cin = c.Cin; a.CinP = c.CinP; a.ld_in = Wp;
                a.w = c.w; a.bias = c.bias; a.CoutP = c.CoutP; a.out_mode = OUT_NHWC;
                if (half == 0) {            // conv1: A -> B = ELU(raw)
                    a.in = A; a.A = B; a.A_elu = 1; a.T = nullptr; a.T_elu = 0;
                    a.in_planes = 0; a.A_planes = 1;
                } else {                    // conv2: B -> trunk (+ residual), next input into A
                    a.in = B; a.resid = T; a.T = T; a.T_elu = last_layer ? 1 : 0;
                    a.A = (last_layer && last_block) ? nullptr : A; a.A_elu = 1;
                    a.in_planes = 1; a.A_planes = (last_layer && last_block) ? -1 : 0;
                    if (last_layer && last_block && tc_head) { a.A_planes = 0; a.A_elu = 0; }     // planes = the trunk itself (already ELU'd)
                }
                prof->begin(c.ks <= 3 ? CAT_CONV_DENSE3 : CAT_CONV_DENSE5, st);     // as conv mode bits 1 / 2
                if (int rc = dispatch_conv(m, np, ROLE_DENSE, c, a, n, st, launches)) return rc;
                prof->end(st);
            }
        }
    }
    {   // heads
        const ConvSlot &c = m->convs[np.head];
        ConvArgs a = {};
        a.in = T; a.in_mode = IN_NHWC; a.Cin = c.Cin; a.CinP = c.CinP; a.ld_in = Wp;
        a.w = c.w; a.bias = c.bias; a.CoutP = c.CoutP;
        a.out_mode = np.out_mode; a.mu = mu; a.scale = scale; a.n_mu = np.n_mu; a.n_sc = np.n_sc;
        a.scale_kind = np.scale_kind; a.out_dim = np.out_dim;
        prof->begin(CAT_CONV_HEAD, st);
        a.in_planes = 0;
        if (int rc = dispatch_conv(m, np, ROLE_HEAD, c, a, n, st, launches)) return rc;
        prof->end(st);
    }
    return BSW_OK;
}

// Test hook: one conv of a loaded model through dispatch_conv, with the epilogue selected by `flags`.  The conv's role
// and net come from the model's plans; a head is named by its mu prefix.  Tensor-core dense convs and heads read plane
// buffer 0, split from in_dev here by the same RNE split the epilogues use; dense convs write plane buffer 1, in-convs
// plane buffer 0.  The written buffer is filled with 0xffff first and copied whole ([2][max_batch,256,Wp], Wp = 64, 128,
// ..., 512) to planes_dev, so rows the conv must not touch can be checked.
extern "C" int bsw_selftest_conv(bsw_model *m, const char *prefix, const float *in_dev, int64_t n, int flags, float *T_dev,
                                 float *A_dev, uint16_t *planes_dev, float *mu_dev, float *scale_dev, void *stream) {
    BSW_REQUIRE(m && prefix && in_dev, "bsw_selftest_conv: null argument");
    BSW_REQUIRE(m->finalized, "model not finalized");
    BSW_REQUIRE(n >= 1 && n <= m->d.max_batch, "batch exceeds the model's max_batch");
    BSW_REQUIRE((flags & ~(BSW_CONV_RESID | BSW_CONV_T | BSW_CONV_T_ELU | BSW_CONV_A | BSW_CONV_A_ELU)) == 0,
                "bsw_selftest_conv: unknown flags");
    auto it = m->names.find(prefix);
    if (it == m->names.end() || it->second.co_off != 0) {
        bsw_set_error("bsw_selftest_conv: '%s' names no conv of this model (heads go by their mu prefix)", prefix);
        return BSW_E_INVALID;
    }
    const int slot = it->second.slot;
    const NetPlan *np = nullptr;
    int role = -1;
    for (const std::vector<NetPlan> *nets : {&m->infer, &m->gen})
        for (const NetPlan &p : *nets) {
            if (p.in_conv == slot) { np = &p; role = ROLE_IN; }
            if (p.head == slot) { np = &p; role = ROLE_HEAD; }
            for (const BlockPlan &bp : p.blocks)
                for (const auto &l : bp.layers)
                    if (l.first == slot || l.second == slot) { np = &p; role = ROLE_DENSE; }
        }
    BSW_REQUIRE(np, "bsw_selftest_conv: the conv is in no net");
    const ConvSlot &c = m->convs[slot];
    cudaStream_t st = (cudaStream_t)stream;
    const size_t plane_bytes = (size_t)m->d.max_batch * 256 * m->Wp * sizeof(uint16_t);
    ConvArgs a = {};
    a.Cin = c.Cin; a.CinP = c.CinP; a.w = c.w; a.bias = c.bias; a.CoutP = c.CoutP;
    a.in = in_dev; a.in_planes = 0; a.A_planes = -1;
    int out_planes = -1, launches = 0;
    if (role == ROLE_HEAD) {
        BSW_REQUIRE(mu_dev && (scale_dev || np->n_sc == 0), "bsw_selftest_conv: head outputs required");
        a.in_mode = IN_NHWC; a.ld_in = m->Wp;
        a.out_mode = np->out_mode; a.mu = mu_dev; a.scale = scale_dev; a.n_mu = np->n_mu; a.n_sc = np->n_sc;
        a.scale_kind = np->scale_kind; a.out_dim = np->out_dim;
        if (head_on_tc(m, *np))
            if (int rc = bsw_tc_split(m, in_dev, 0, n, st)) return rc;
    } else {
        BSW_REQUIRE(T_dev || !(flags & (BSW_CONV_RESID | BSW_CONV_T)), "bsw_selftest_conv: T_dev required");
        a.out_mode = OUT_NHWC;
        a.resid = (flags & BSW_CONV_RESID) ? T_dev : nullptr;           // in place, as run_net does
        a.T = (flags & BSW_CONV_T) ? T_dev : nullptr; a.T_elu = (flags & BSW_CONV_T_ELU) ? 1 : 0;
        a.A = (flags & BSW_CONV_A) ? (A_dev ? A_dev : m->bufA) : nullptr; a.A_elu = (flags & BSW_CONV_A_ELU) ? 1 : 0;
        if (role == ROLE_IN) {
            a.in_mode = np->in_mode; a.in_dim = np->in_dim; a.ld_in = 0;
            if (in_writes_planes(m, *np)) {
                BSW_REQUIRE(flags & BSW_CONV_A, "bsw_selftest_conv: this in-conv writes the first layer's input (BSW_CONV_A)");
                out_planes = 0;
            }
        } else {
            a.in_mode = IN_NHWC; a.ld_in = m->Wp;
            if (net_on_tc(m)) {
                if (int rc = bsw_tc_split(m, in_dev, 0, n, st)) return rc;
                if (flags & BSW_CONV_A) out_planes = a.A_planes = 1;
            }
        }
    }
    void *hi = nullptr, *lo = nullptr;
    if (out_planes >= 0) {
        BSW_REQUIRE(planes_dev, "bsw_selftest_conv: planes_dev required on the tensor-core path");
        bsw_tc_planes(m, out_planes, &hi, &lo);
        BSW_CUDA(cudaMemsetAsync(hi, 0xff, plane_bytes, st));
        BSW_CUDA(cudaMemsetAsync(lo, 0xff, plane_bytes, st));
    }
    if (int rc = dispatch_conv(m, *np, role, c, a, n, st, &launches)) return rc;
    if (out_planes >= 0) {
        BSW_CUDA(cudaMemcpyAsync(planes_dev, hi, plane_bytes, cudaMemcpyDeviceToDevice, st));
        BSW_CUDA(cudaMemcpyAsync((char *)planes_dev + plane_bytes, lo, plane_bytes, cudaMemcpyDeviceToDevice, st));
    }
    return BSW_OK;
}

int bsw_model_run(bsw_model *m, bool infer, int level, const float *given, int64_t n, float *mu, float *scale,
                  int scale_per_stream, cudaStream_t st, int *launches, BswProf *prof) {
    BSW_REQUIRE(m && given && mu, "bsw_vae: null argument");
    BSW_REQUIRE(level >= 0 && level < m->d.nz, "bsw_vae: level out of range");
    const NetPlan &np = infer ? m->infer[level] : m->gen[level];
    int dummy = 0;
    if (!launches) launches = &dummy;
    BSW_REQUIRE(scale || np.n_sc == 0, "bsw_vae: scale output required");
    if (int rc = run_net(m, np, given, n, mu, scale, st, launches, prof)) return rc;
    if (!infer && level == 0 && !m->d.cond_xscale && scale) {
        int64_t rows = scale_per_stream ? n : 1;
        if (prof) prof->begin(CAT_MISC, st);
        k_broadcast_rows<<<(unsigned)((rows * m->xdim + 255) / 256), 256, 0, st>>>(m->xscale, scale, m->xdim, rows);
        BSW_LAUNCH_CHECK();
        if (prof) prof->end(st);
        ++*launches;
    }
    return BSW_OK;
}

extern "C" int bsw_vae_infer(bsw_model *m, int level, const float *given, int64_t n, float *mu, float *scale, void *stream) {
    return bsw_model_run(m, true, level, given, n, mu, scale, 1, (cudaStream_t)stream, nullptr);
}
extern "C" int bsw_vae_generate(bsw_model *m, int level, const float *given, int64_t n, float *mu, float *scale,
                                int scale_per_stream, void *stream) {
    return bsw_model_run(m, false, level, given, n, mu, scale, scale_per_stream, (cudaStream_t)stream, nullptr);
}
