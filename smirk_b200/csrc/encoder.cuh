// The encoder handle shared by the eval path (encoder.cu) and the train-mode path (encoder_train.cu): the MobileNetV3
// "minimal" layer lists, the per-backbone topology, and the fork/join walk over the backbones.
#pragma once
#include "common.cuh"

namespace enc {

struct ConvW { float* w = nullptr; float* wt = nullptr; float* wt_lo = nullptr; float* scale = nullptr; float* bias = nullptr; int cin = 0, cout = 0; };   // w: [K][N] fp32 path, wt: [N][K] tensor-core path (TF32 heads), wt_lo: TF32 tails (3xTF32 path)
enum Kind { DS = 0, IR = 1, CN = 2 };
struct BlockDef { Kind kind; int stride; float exp; int cout; };
// pw_f32: fp32 [K][N] copy of a DS block's 1x1 (fused stem path).  *_d: dgrad weights (see fold_conv).
// sv_a / sv_b: saved-tensor indices of the block's ReLU outputs (IR: expand, depthwise; DS: depthwise; CN: its output).
// Train handles only: sv_z[j] the pre-BN output of the block's j-th conv, sv_out the block output (DS / IR), bn0 the
// index of the block's first BatchNorm within its backbone.
struct Block { Kind kind; int stride, cin, mid, cout; bool skip; ConvW pw, dw, pwl; ConvW pw_f32; ConvW pw_d, dw_d, pwl_d; int sv_a = -1, sv_b = -1;
               int sv_z[3] = {-1, -1, -1}, sv_out = -1, bn0 = 0; };

struct Backbone {
    ConvW stem, stem_d;
    std::vector<Block> blocks;
    int feat = 0;
    float *head_w = nullptr, *head_b = nullptr;
    int n_out = 0;
    uint8_t* codes = nullptr;
    int sv_stem = -1, sv_head = -1;
    int sv_zstem = -1, sv_pool = -1;           // train handles: the stem's pre-BN output, the pooled features [B, feat]
    size_t max_act = 0;                        // floats per image of the largest activation
};

constexpr BlockDef kLarge[] = {
    {DS, 1, 1.f, 16},
    {IR, 2, 4.f, 24}, {IR, 1, 3.f, 24},
    {IR, 2, 3.f, 40}, {IR, 1, 3.f, 40}, {IR, 1, 3.f, 40},
    {IR, 2, 6.f, 80}, {IR, 1, 2.5f, 80}, {IR, 1, 2.3f, 80}, {IR, 1, 2.3f, 80},
    {IR, 1, 6.f, 112}, {IR, 1, 6.f, 112},
    {IR, 2, 6.f, 160}, {IR, 1, 6.f, 160}, {IR, 1, 6.f, 160},
    {CN, 1, 1.f, 960}};
constexpr BlockDef kSmall[] = {
    {DS, 2, 1.f, 16},
    {IR, 2, 4.5f, 24}, {IR, 1, 3.67f, 24},
    {IR, 2, 4.f, 40}, {IR, 1, 6.f, 40}, {IR, 1, 6.f, 40},
    {IR, 1, 3.f, 48}, {IR, 1, 3.f, 48},
    {IR, 2, 6.f, 96}, {IR, 1, 6.f, 96}, {IR, 1, 6.f, 96},
    {CN, 1, 1.f, 576}};
// Blocks per stage (the module paths blocks.<stage>.<i>) and the reference's module names of the backbones and heads.
constexpr int kStageLarge[] = {1, 2, 3, 4, 2, 3, 1}, kStageSmall[] = {1, 2, 3, 2, 3, 1};
constexpr const char* kEncName[3] = {"pose_encoder", "shape_encoder", "expression_encoder"};
constexpr const char* kHeadName[3] = {"pose_cam_layers.0", "shape_layers.0", "expression_layers.0"};

inline int make_divisible(double v, int divisor = 8) {
    int nv = std::max(divisor, (int)(v + divisor / 2.0) / divisor * divisor);
    if (nv < 0.9 * v) nv += divisor;
    return nv;
}

}  // namespace enc

struct SmkEncoder {
    enc::Backbone bb[3];
    int n_shape = 300, n_exp = 50, precision = 0;
    size_t max_act = 0;          // floats per image of the largest activation
    bool fuse_xdw = false;       // precision >= 2: inverted-residual blocks use the fused expand+depthwise kernel
    bool x3 = false;             // precision 3: 3xTF32 error-compensated tensor-core arithmetic (fp32-equivalent), no TF32 rounding of activations
    bool train = false;          // a train-mode handle (smk_encoder_train_create): topology only, no packed weights
    size_t stats_floats = 0;     // train handles: floats of BatchNorm statistics after the saved tensors (mean, invstd per BN)
    bool present[3] = {false, false, false};   // a handle may hold a subset of the backbones (PoseEncoder / ShapeEncoder / ExpressionEncoder alone)
    float *ones = nullptr, *zeros = nullptr;   // unit scale / zero bias of the dgrad GEMM epilogues
    smk::SavedLayout saved;                    // of the grad-mode forward: forward order within a backbone, backbones in slot order
    smk::DeviceArena arena;
    // Fork/join plumbing for running the backbones as parallel branches of the caller's stream.  A forward takes the
    // next set of a small pool (atomic round-robin), so up to kForkSets forwards of one handle may be in flight on
    // different streams (with distinct workspaces) without sharing an event or a side stream: the handle is re-entrant.
    static constexpr int kForkSets = 8;
    struct ForkSet { cudaStream_t side[2] = {nullptr, nullptr}; cudaEvent_t fork = nullptr, join[2] = {nullptr, nullptr}; };
    ForkSet forks[kForkSets];
    mutable unsigned next_fork = 0;
    ~SmkEncoder() {
        for (auto& f : forks) {
            for (int s = 0; s < 2; ++s) { if (f.side[s]) cudaStreamDestroy(f.side[s]); if (f.join[s]) cudaEventDestroy(f.join[s]); }
            if (f.fork) cudaEventDestroy(f.fork);
        }
    }
};

namespace enc {

// The handle's side streams and events; -> cudaSuccess or the first error.
inline cudaError_t create_forks(SmkEncoder* h) {
    cudaError_t e = cudaSuccess;
    for (auto& f : h->forks) {
        for (int s = 0; s < 2 && e == cudaSuccess; ++s) {
            e = cudaStreamCreateWithFlags(&f.side[s], cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f.join[s], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f.fork, cudaEventDisableTiming);
    }
    return e;
}

// One unit of work: n = 1 backbone, or the pair idx = {1, 2}, on stream st.
struct Unit { int n; int idx[2]; cudaStream_t st; };

// Runs run(unit) (-> status; the first error stops the walk) over the backbones with use[i] set.  The three backbones
// are independent (smirk_encoder.py:123-133 merely runs them one after another): with more than one in use, the units
// fork from main_st onto the side streams of one of the handle's fork sets, so their many small, latency-bound layers
// overlap, and join back into main_st — even after an error, so a capturing stream is left consistent.  Event
// record/wait on other streams is legal under stream capture, so a CUDA graph of the caller's stream gets parallel
// branches.  The two "large" backbones (shape, expression) have the same layer list, so on the eval tensor-core path they
// advance in lock step as one unit and every layer of the pair is ONE launch; the small (pose) backbone is its own unit.
// A train handle runs every backbone as its own unit.
template <typename Run>
int for_each_unit(const SmkEncoder* h, const bool use[3], cudaStream_t main_st, const char* what, Run&& run) {
    const int n_use = (int)use[0] + (int)use[1] + (int)use[2];
    const bool concurrent = !smk::profiling() && n_use > 1;       // the event profiler wants one kernel at a time
    const SmkEncoder::ForkSet& fk = h->forks[__atomic_fetch_add(&h->next_fork, 1u, __ATOMIC_RELAXED) % SmkEncoder::kForkSets];
    Unit units[3]; int n_units = 0;
    if (use[0]) units[n_units++] = Unit{1, {0, 0}, main_st};
    if (!h->train && h->precision >= 1 && use[1] && use[2]) units[n_units++] = Unit{2, {1, 2}, concurrent ? fk.side[0] : main_st};
    else for (int i = 1; i < 3; ++i) if (use[i]) units[n_units++] = Unit{1, {i, i}, concurrent ? fk.side[i - 1] : main_st};
    if (!use[0] && n_units > 0) units[0].st = main_st;                             // without pose, the first unit takes the caller's stream
    if (concurrent) {
        SMK_CHECK_CUDA(cudaEventRecord(fk.fork, main_st));
        for (int s = 0; s < 2; ++s) SMK_CHECK_CUDA(cudaStreamWaitEvent(fk.side[s], fk.fork, 0));
    }
    int rc = 0;
    for (int u = 0; u < n_units && !rc; ++u) rc = run(units[u]);
    for (int s = 0; s < 2 && concurrent; ++s) {
        cudaError_t e1 = cudaEventRecord(fk.join[s], fk.side[s]);
        cudaError_t e2 = e1 == cudaSuccess ? cudaStreamWaitEvent(main_st, fk.join[s], 0) : e1;
        if (!rc && e2 != cudaSuccess) { smk::set_error("%s: stream join failed: %s", what, cudaGetErrorString(e2)); rc = (int)e2; }
    }
    return rc;
}

// Stem dgrad of the input gradient: sums the backbones' stem pre-activation gradients g[i] [B,112,112,16] (null: skipped)
// through their stem weights w[i] [27][16] into the NCHW image gradient (zero when every g is null).  encoder.cu.
int stem_dgrad(const float* const g[3], const float* const w[3], int B, float* g_img, cudaStream_t st);

}  // namespace enc
