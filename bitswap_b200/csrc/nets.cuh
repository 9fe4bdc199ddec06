// Internal declarations of the VAE runtime (shared by nets.cu, conv_tc.cu, codec.cu).
#pragma once
#include <map>
#include <string>
#include <vector>
#include "bsw_common.cuh"

enum { IN_NHWC = 0, IN_CHW_Z = 1, IN_CHW_X = 2 };
enum { OUT_NHWC = 0, OUT_HEAD_Z = 1, OUT_HEAD_X = 2 };
enum { SCALE_NONE = 0, SCALE_INFER = 1, SCALE_DEEPGEN = 2, SCALE_X = 3 };

struct ConvArgs {
    // input
    const float *in;      // IN_NHWC: [n,256,ld_in] ; IN_CHW_*: flat `given` [n,in_dim]
    int in_mode, in_dim, Cin, CinP, ld_in;
    // weights [taps][CinP][CoutP] (weight norm folded), bias [CoutP]
    const float *w, *bias;
    int CoutP;
    // hidden-layer epilogue: r = conv + bias (+ resid); T = T_elu ? ELU(r) : r; A = A_elu ? ELU(T) : T
    int out_mode;
    const float *resid;
    float *T, *A;
    int T_elu, A_elu;
    // tensor-core path: index (0/1) of the bf16 hi/lo plane buffer read / written as the conv input (-1: none)
    int in_planes, A_planes;
    // head epilogue
    float *mu, *scale;
    int n_mu, n_sc, scale_kind, out_dim;
};

struct ConvSlot {
    std::string name;
    int Cin, Cout, ks, CinP, CoutP;
    float *w, *bias;                 // device, SIMT layout
    std::vector<float> host_w, host_b;
    int loaded_mask, parts;
    // tensor-core path (conv_tc.cu): bf16 hi/lo weight planes [taps][CoutP][CinP], K-major
    void *w_hi = nullptr, *w_lo = nullptr;
    int tc_index = -1;
};
struct NameRef { int slot, co_off; };
struct BlockPlan { std::vector<std::pair<int, int>> layers; };
struct NetPlan {
    int in_conv, in_mode, in_dim;
    std::vector<BlockPlan> blocks;
    int head, out_mode, n_mu, n_sc, scale_kind, out_dim;
};

struct bsw_model {
    bsw_model_desc d;
    int Wp, zdim, xdim;
    std::vector<ConvSlot> convs;
    std::map<std::string, NameRef> names;
    std::vector<NetPlan> infer, gen;
    float *bufT, *bufA, *bufB;       // [max_batch, 256, Wp] float32: trunk + two conv-input buffers
    float *xscale;                   // [xdim] unconditional x-scale
    bool have_gen_std, finalized;
    bool tc_ready = false;
    int tc_precision = BSW_TC_SPLIT; // arithmetic of the tensor-core convs (bsw_model_set_tc_precision)
    void *tc_state = nullptr;        // owned by conv_tc.cu
    void *tc_slots = nullptr;
    bool digest_ok = false;          // digest holds bsw_model_digest of the weights loaded now (digest.cu)
    uint32_t digest[4];
};

// Per-kernel-category device timing (CUDA events on the launching stream), used by bench.py's roofline.
enum { CAT_MISC = 0, CAT_CONV_IN = 1, CAT_CONV_DENSE3 = 2, CAT_CONV_DENSE5 = 3, CAT_CONV_HEAD = 4, CAT_POP_Z = 5,
       CAT_PUSH_Z = 6, CAT_POP_X = 7, CAT_PUSH_X = 8, CAT_PRIOR = 9, CAT_ROWS_Z = 10, CAT_ROWS_X = 11, CAT_COUNT = 12 };
struct BswProf {
    bool on = false;
    std::vector<cudaEvent_t> pool;
    std::vector<int> cats;          // category of event pair i (events 2i, 2i+1)
    size_t used = 0;
    double ms[CAT_COUNT] = {0};
    int64_t n[CAT_COUNT] = {0};
    void begin(int cat, cudaStream_t st) {
        if (!on) return;
        if (used + 2 > pool.size()) {
            cudaEvent_t a, b;
            cudaEventCreate(&a); cudaEventCreate(&b);
            pool.push_back(a); pool.push_back(b);
        }
        cats.push_back(cat);
        cudaEventRecord(pool[used], st);
    }
    void end(cudaStream_t st) {
        if (!on) return;
        cudaEventRecord(pool[used + 1], st);
        used += 2;
    }
    void collect() {          // synchronises on the last event
        if (used) cudaEventSynchronize(pool[used - 1]);
        for (size_t i = 0; i < used / 2; ++i) {
            float t = 0.f;
            cudaEventElapsedTime(&t, pool[2 * i], pool[2 * i + 1]);
            ms[cats[i]] += t; n[cats[i]] += 1;
        }
        used = 0; cats.clear();
    }
    void reset() { collect(); for (int i = 0; i < CAT_COUNT; ++i) { ms[i] = 0; n[i] = 0; } }
};

int bsw_conv_simt(const ConvArgs &a, int ks, int64_t n, cudaStream_t st);
int bsw_model_run(bsw_model *m, bool infer, int level, const float *given, int64_t n, float *mu, float *scale,
                  int scale_per_stream, cudaStream_t st, int *launches, BswProf *prof = nullptr);
// conv_tc.cu
int bsw_model_tc_prepare(bsw_model *m);
void bsw_model_tc_release(bsw_model *m);
int bsw_conv_tc(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st);
bool bsw_conv_tc_head_available(bsw_model *m, const ConvSlot &c);
int bsw_model_tc_heads(bsw_model *m);
int bsw_conv_tc_head(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st);
int bsw_tc_split(bsw_model *m, const float *in, int which, int64_t n, cudaStream_t st);
void bsw_tc_planes(bsw_model *m, int which, void **hi, void **lo);
int bsw_conv_tc_in(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st, int *launches);
