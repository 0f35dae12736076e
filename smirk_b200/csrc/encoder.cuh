// The encoder handle shared by the eval path (encoder.cu) and the train-mode path (encoder_train.cu): the MobileNetV3
// "minimal" layer lists, the per-backbone topology and its one builder, and the fork/join walk over the backbones.
#pragma once
#include "train_common.cuh"
#include <string>

namespace enc {

// A conv with its folded BatchNorm.  fwd / dgrad: the weights of the forward and of the input gradient (see fold_conv): a 1x1
// conv's are smk::conv operands, a depthwise or stem conv's are fp32 in fwd.w / dgrad.w, in layouts of their own.
struct ConvW { smk::GemmW fwd{}, dgrad{}; float* scale = nullptr; float* bias = nullptr; int cin = 0, cout = 0; };
enum Kind { DS = 0, IR = 1, CN = 2 };
struct BlockDef { Kind kind; int stride; float exp; int cout; };
// path: the block's module path, <encoder>.encoder.blocks.<stage>.<i>; hin / hout: input / output resolution.
// sv_a / sv_b: saved-tensor indices of the block's ReLU outputs (IR: expand, depthwise; DS: depthwise; CN: its output); eval handles.
struct Block { Kind kind; int stride, cin, mid, cout; bool skip; std::string path; int hin, hout;
               ConvW pw, dw, pwl; int sv_a = -1, sv_b = -1; };

// Train handles walk a backbone as a flat list, in forward order, of conv + BatchNorm (+ skip) (+ ReLU) layers.  The stem is
// entry 0, so the index is the BatchNorm's index in the tensor list (5 tensors per entry, one num_batches_tracked).
enum Op { STEM, PW, DW };
struct Layer {
    Op op; int cin, cout, stride, hin, hout;
    int sv_in, sv_z, sv_y;   // saved-tensor indices of the input (-1: the image), the pre-BN output, the BN (+ skip, ReLU) output
    bool relu;               // ReLU after the BatchNorm
    bool first;              // first layer of its block
    int skip;                // last layer of a block with a skip connection: saved index of the block input; otherwise -1
    size_t stats;            // offset in floats, within the handle's statistics area, of mean[cout]; invstd[cout] follows
    int pw;                  // PW: index among the backbone's 1x1 convs (its slot of the per-call weight pack); otherwise -1
};

struct Backbone {
    ConvW stem;
    std::vector<Block> blocks;
    std::vector<Layer> layers;                 // train handles
    int feat = 0;
    float *head_w = nullptr, *head_b = nullptr;
    int n_out = 0;
    uint8_t* codes = nullptr;
    int sv_stem = -1, sv_head = -1;            // sv_stem: eval handles (a train handle's is layers[0].sv_y)
    int sv_pool = -1;                          // train handles: the pooled features [B, feat]
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
    bool live = false;           // a live eval handle (smk_encoder_live_create): weights set on the device by smk_encoder_refresh
    bool refreshed = false;      // live handles: refreshed at least once
    trn::LivePlan plan;          // live handles: the refresh's folds and pack jobs (lists = backbones)
    int live_tensors[3] = {0, 0, 0};           // live handles: tensors per backbone the refresh reads
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

// Everything about backbone i that follows from its layer list and the head widths: the blocks (channels, resolutions,
// module paths), feat, n_out and the activation sizes.  Weights and saved tensors are the caller's.
inline void build_backbone(SmkEncoder* h, int i) {
    Backbone& bb = h->bb[i];
    const BlockDef* defs = i == 0 ? kSmall : kLarge;
    const int nb = i == 0 ? (int)(sizeof(kSmall) / sizeof(BlockDef)) : (int)(sizeof(kLarge) / sizeof(BlockDef));
    const int* stages = i == 0 ? kStageSmall : kStageLarge;
    int cin = 16, res = 112, stage = 0, in_stage = 0;
    bb.max_act = (size_t)112 * 112 * 16;
    for (int k = 0; k < nb; ++k) {
        Block b{};
        b.kind = defs[k].kind; b.stride = defs[k].stride; b.cin = cin; b.cout = defs[k].cout;
        b.skip = b.kind != CN && b.stride == 1 && b.cin == b.cout;
        b.mid = b.kind == IR ? make_divisible((double)cin * defs[k].exp) : cin;
        b.hin = res; b.hout = (res + b.stride - 1) / b.stride;
        b.path = std::string(kEncName[i]) + ".encoder.blocks." + std::to_string(stage) + "." + std::to_string(in_stage);
        if (++in_stage == stages[stage]) { ++stage; in_stage = 0; }
        bb.max_act = std::max(bb.max_act, (size_t)b.hin * b.hin * b.mid);           // expanded tensor at input resolution
        bb.max_act = std::max(bb.max_act, (size_t)b.hout * b.hout * std::max(b.mid, b.cout));
        res = b.hout; cin = b.cout;
        bb.blocks.push_back(b);
    }
    bb.feat = cin;
    bb.n_out = i == 0 ? 6 : i == 1 ? h->n_shape : h->n_exp + 5;
    h->max_act = std::max(h->max_act, bb.max_act);
}

// The device state every handle has besides its layers: the expression head's clamp codes (smirk_encoder.py:105-108), the
// unit scale / zero bias of the dgrad GEMM epilogues, and the fork/join streams and events; -> cudaSuccess or the first error.
inline cudaError_t finish_create(SmkEncoder* h) {
    cudaError_t e = cudaSuccess;
    if (h->present[2]) {
        const int ne = h->n_exp;
        std::vector<uint8_t> codes(h->bb[2].n_out, 0);
        codes[ne] = codes[ne + 1] = 1; codes[ne + 2] = 2; codes[ne + 3] = codes[ne + 4] = 3;
        e = h->arena.upload(codes, &h->bb[2].codes);
    }
    std::vector<float> ones(1024, 1.f), zeros(1024, 0.f);
    if (e == cudaSuccess) e = h->arena.upload(ones, &h->ones);
    if (e == cudaSuccess) e = h->arena.upload(zeros, &h->zeros);
    return e == cudaSuccess ? create_forks(h) : e;
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
